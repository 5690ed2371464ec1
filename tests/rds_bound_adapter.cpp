// tests/rds_bound_adapter.cpp -- dsp::b200::FrontEnd with one WFM VFO and the radio's "Decode RDS" (bindRDS) as worker-thread
// blocks: every chunk's audio and RDS records are read from the two output streams.  Writes the decoded bits (one byte each)
// and prints "<chunks> <audio samples> <symbols>".  Built and run by tests/test_gpu_rds_bound.py.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "dsp/b200/frontend.h"

int main(int argc, char** argv) {
    if (argc < 5) { fprintf(stderr, "usage: %s iq.f32 bits_out.u8 samplerate offset\n", argv[0]); return 2; }
    if (b200_init(0) != 0) { fprintf(stderr, "%s\n", b200_last_error()); return 3; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { return 2; }
    fseek(f, 0, SEEK_END);
    long bytes = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<dsp::complex_t> iq(bytes / sizeof(dsp::complex_t));
    if (fread(iq.data(), sizeof(dsp::complex_t), iq.size(), f) != iq.size()) { return 2; }
    fclose(f);

    const double fs = atof(argv[3]);
    const int chunk = 40000;                       // 100 samples of the 5 kS/s branch: every chunk carries symbols
    const size_t nch = iq.size() / chunk;
    dsp::stream<dsp::complex_t> input(chunk);
    dsp::b200::FrontEnd fe;
    fe.init(&input, fs, 0, 20.0, B200_WIN_NUTTALL, nullptr, nullptr, nullptr);
    b200_vfo_cfg cfg = {};
    cfg.offset = atof(argv[4]); cfg.out_samplerate = 250000.0; cfg.bandwidth = 150000.0; cfg.demod = B200_DEMOD_WFM_STEREO;
    cfg.deviation = 75000.0; cfg.low_pass = 1;
    int id = fe.addVFO(cfg);
    int rid = id >= 0 ? fe.bindRDS(id) : -1;
    if (rid < 0) { fprintf(stderr, "%s\n", b200_last_error()); return 3; }
    fe.start();
    std::vector<unsigned char> bits;
    size_t audio = 0, chunks = 0;
    for (size_t k = 0; k < nch; k++) {
        memcpy(input.writeBuf, &iq[k * chunk], chunk * sizeof(dsp::complex_t));
        if (!input.swap(chunk)) { break; }
        // the worker swaps its outputs in id order: the audio, then the records
        int n = fe.vfoOut(id)->read();
        if (n <= 0) { break; }
        audio += (size_t)n;
        fe.vfoOut(id)->flush();
        int m = fe.vfoOut(rid)->read();
        if (m <= 0) { break; }
        const b200_rds_symbol* r = dsp::b200::FrontEnd::rdsSymbols(fe.vfoOut(rid));
        for (int i = 0; i < m; i++) { bits.push_back((unsigned char)r[i].bit); }
        fe.vfoOut(rid)->flush();
        chunks++;
    }
    fe.stop();
    fe.removeVFO(id);                              // unbinds the RDS output first
    FILE* o = fopen(argv[2], "wb");
    if (!o) { return 2; }
    fwrite(bits.data(), 1, bits.size(), o);
    fclose(o);
    printf("%zu %zu %zu\n", chunks, audio, bits.size());
    return chunks == nch ? 0 : 4;
}

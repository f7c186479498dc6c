// r8b::CDSPResamplerBatch::setDither through the C++ front: one batch of two channels, channel 1 set to 9-tap shaped
// TPDF, fed one block of a fp64 input file and converted to int16 on the device; writes the fp64 twin output and the
// int16 output (count, then samples, per channel) so the caller can check the bytes against the host quantiser.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "r8b/CDSPResampler.h"

int main(int argc, char** argv)
{
    if (argc != 4) return 2;
    const int frames = atoi(argv[3]), n_ch = 2;
    std::vector<double> in((size_t) n_ch * frames);
    FILE* f = fopen(argv[1], "rb");
    if (!f || fread(in.data(), sizeof(double), in.size(), f) != in.size()) return 3;
    fclose(f);
    r8b::CDSPResamplerBatch dith(n_ch, 44100.0, 48000.0, frames, 2.0, 180.15, r8b::fprLinearPhase, 0);
    r8b::CDSPResamplerBatch twin(n_ch, 44100.0, 48000.0, frames, 2.0, 180.15, r8b::fprLinearPhase, 0);
    r8bgpu_dither cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.kind = R8BGPU_DITHER_TPDF;
    cfg.seed = 12345;
    cfg.n_taps = 9;
    const double taps[9] = {2.033, -2.165, 1.959, -1.590, 0.6149, -0.2, 0.1, -0.05, 0.01};
    for (int k = 0; k < 9; k++) cfg.taps[k] = taps[k];
    const int ch = 1;
    if (dith.setDither(&ch, 1, &cfg) != 0) return 4;
    r8bgpu_dither bad = cfg;
    bad.kind = 7;
    if (dith.setDither(&ch, 1, &bad) == 0) return 5; // refused
    const int cap = twin.getMaxOutLen();
    std::vector<double> y((size_t) n_ch * cap);
    std::vector<short> q((size_t) n_ch * cap);
    const int n = twin.process(in.data(), (size_t) frames, frames, y.data(), (size_t) cap, cap);
    r8bgpu_buffer bi = {in.data(), R8BGPU_F64, 0, (size_t) frames, 1.0};
    r8bgpu_buffer bo = {q.data(), R8BGPU_S16, 0, (size_t) cap, 32767.0};
    const int m = r8bgpu_batch_process_host_fmt(dith.handle(), &bi, frames, &bo, cap);
    if (n < 0 || m != n) return 6;
    f = fopen(argv[2], "wb");
    for (int c = 0; c < n_ch; c++) {
        const long long k = n;
        fwrite(&k, sizeof k, 1, f);
        fwrite(&y[(size_t) c * cap], sizeof(double), (size_t) n, f);
        fwrite(&q[(size_t) c * cap], sizeof(short), (size_t) n, f);
    }
    fclose(f);
    printf("%d\n", n);
    return 0;
}

// tests/cpp/oneshot_crops_demo.cpp -- CDSPResamplerBatch::oneshotCrops, both overloads, on two clips of exactly
// representable samples.  Each crop's output is printed as one line "<name> <crop> <hex floats...>"; a failed call
// prints "<name> -1 <last error>".
#include <cstdio>
#include <vector>

#include "r8b/CDSPResampler.h"

static const int N = 20000;

static double sample(int r, int i) { return (double) ((i * 7 + r * 3) % 101 - 50) / 64.0; }

static void run(const char* name, int rc, const std::vector<double>& out, const r8bgpu_crop* crops, int n_crops, int stride)
{
    if (rc != 0) {
        printf("%s -1 %s\n", name, r8bgpu_last_error());
        return;
    }
    for (int k = 0; k < n_crops; k++) {
        printf("%s %d", name, k);
        for (long long i = 0; i < crops[k].o1 - crops[k].o0; i++) printf(" %a", out[(size_t) k * stride + (size_t) i]);
        printf("\n");
    }
}

int main()
{
    std::vector<double> in(2 * N);
    for (int r = 0; r < 2; r++)
        for (int i = 0; i < N; i++) in[(size_t) r * N + i] = sample(r, i);
    const long long lens[2] = {N, 15000};
    const r8bgpu_crop crops[3] = {{1, 0, 100, 160}, {0, 0, 2000, 2100}, {0, 0, 6000, 6060}};
    const int stride = 100;
    {
        r8b::CDSPResamplerBatch b(4, 48000.0, 16000.0, 4096, 2.0, 206.91);
        std::vector<double> out(3 * stride, 0.0);
        run("one_pair", b.oneshotCrops(&in[0], N, 2, lens, NULL, 3, crops, &out[0], stride), out, crops, 3, stride);
    }
    {
        const double src[4] = {48000.0, 48000.0, 44100.0, 44100.0}, dst[4] = {16000.0, 16000.0, 16000.0, 16000.0};
        r8b::CDSPResamplerBatch b(4, src, dst, 4096, 2.0, 206.91);
        const double csrc[2] = {44100.0, 48000.0}, cdst[2] = {16000.0, 16000.0};
        std::vector<double> out(3 * stride, 0.0);
        run("per_clip", b.oneshotCrops(&in[0], N, 2, csrc, cdst, lens, NULL, 3, crops, &out[0], stride), out, crops, 3,
            stride);
    }
    return 0;
}

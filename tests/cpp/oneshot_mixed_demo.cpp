// tests/cpp/oneshot_mixed_demo.cpp -- the per-clip-rate overloads of CDSPResamplerBatch::oneshotLong /
// oneshotLongAdjoint and the r8bgpu_batch_oneshot_mixed* entry points, called once each.  Each line of the output is
// "<name> <return code> <last error, or '-'>".
#include <cstdio>
#include <vector>

#include "r8b/CDSPResampler.h"

static void report(const char* name, int rc)
{
    const char* e = r8bgpu_last_error();
    printf("%s %d %s\n", name, rc, rc != 0 && e != NULL && e[0] != 0 ? e : "-");
}

int main()
{
    const double src[3] = {44100.0, 16000.0, 44100.0}, dst[3] = {16000.0, 16000.0, 16000.0};
    r8b::CDSPResamplerBatch b(3, src, dst, 4096, 2.0, 206.91);
    // two clips at the batch's two rate pairs
    const double csrc[2] = {16000.0, 44100.0}, cdst[2] = {16000.0, 16000.0};
    const long long lens[2] = {3000, 5000};
    std::vector<double> in(2 * 5000, 0.25), out(2 * 5000, 0.0);
    report("long", b.oneshotLong(&in[0], 5000, 2, csrc, cdst, lens, &out[0], 5000, NULL));
    // a rate pair the batch has no channel for
    const double usrc[1] = {48000.0}, udst[1] = {16000.0};
    report("long_unknown_pair", b.oneshotLong(&in[0], 5000, 1, usrc, udst, lens, &out[0], 5000, NULL));
    report("adjoint_unknown_pair", b.oneshotLongAdjoint(NULL, 5000, 1, usrc, udst, lens, NULL, NULL, 5000));
    // the C entry points without a batch
    r8bgpu_buffer bi = {&in[0], R8BGPU_F64, 0, 5000, 1.0}, bo = {&out[0], R8BGPU_F64, 0, 5000, 1.0};
    const int po[2] = {0, 1};
    report("c_mixed", r8bgpu_batch_oneshot_mixed(NULL, &bi, 2, po, lens, &bo, NULL, NULL));
    report("c_mixed_host", r8bgpu_batch_oneshot_mixed_host(NULL, &bi, 2, po, lens, &bo, NULL, NULL));
    report("c_adjoint_mixed", r8bgpu_batch_oneshot_adjoint_mixed(NULL, &bo, 2, po, lens, NULL, &bi));
    return 0;
}

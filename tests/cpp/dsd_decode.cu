// Host build of the DSD decode (r8b_dsd.cuh) for tests/test_dsd_cpu.py: samples [i0, i0 + n) of channel c of a planar
// (byte row c at c*stride) or interleaved (byte frame f at f*stride, channel c at +c) DSD buffer, as the device reads them.
#include "../../r8brain-free-src_b200/csrc/r8b_dsd.cuh"

extern "C" void dsd_decode(const unsigned char* raw, int interleaved, long long stride, int c, long long i0, long long n, int msb,
                           double scale, double* out)
{
    for (long long k = 0; k < n; k++) {
        const long long i = i0 + k;
        out[k] = interleaved ? r8bgpu::dsd_value(raw[(i >> 3) * stride + c], i, msb != 0, scale)
                             : r8bgpu::dsd_load(raw + c * stride, i, msb != 0, scale);
    }
}

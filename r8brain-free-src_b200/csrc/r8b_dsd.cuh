// r8b_dsd.cuh -- the one-bit DSD input formats (include/r8bgpu.h, "caller-side sample formats"): R8BGPU_DSD_LSB (DSF bit
// order, bit 0 of a byte is the earliest sample) and R8BGPU_DSD_MSB (DSDIFF, bit 7 first).  A bit is +scale (1) or -scale
// (0): exact, and the same value as __dmul_rn(+-1.0, scale), the rule of every other input format.  __host__ __device__,
// so the conversion kernels (r8b_format_dsd.cu), the half-band decimators that decode in their loads and the history copy
// (r8b_kernels.cu) and the host test of the layout all take their bits from this one module.
#pragma once
#include "r8b_fft.cuh"
#include "r8b_kernels.h"

namespace r8bgpu {

R8B_HD bool is_dsd_format(int fmt) { return fmt == FMT_DSD_LSB || fmt == FMT_DSD_MSB; }

// Sample i of a row of DSD bytes (i counted from the row's first sample).
R8B_HD double dsd_value(unsigned char byte, long long i, bool msb, double scale)
{
    const int k = (int) (i & 7);
    return ((byte >> (msb ? 7 - k : k)) & 1) ? scale : -scale;
}

R8B_HD double dsd_load(const unsigned char* row, long long i, bool msb, double scale)
{
    return dsd_value(R8B_LDG(row + (i >> 3)), i, msb, scale);
}

} // namespace r8bgpu

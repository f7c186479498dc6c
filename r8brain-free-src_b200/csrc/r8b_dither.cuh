// r8b_dither.cuh -- the dithered quantiser of integer outputs (include/r8bgpu.h, "dithered integer output"): TPDF noise
// from a counter-based generator and error-feedback noise shaping.  Plain arithmetic with every rounding spelled out, so
// the device kernel (k_dither_shape, r8b_format.cu) and the host pin (r8bgpu_dither_quantize_host) produce the same bits.
#pragma once
#include <cfloat>

#include "../../include/r8bgpu.h"
#include "r8b_fft.cuh"
#include "r8b_kernels.h"

namespace r8bgpu {

constexpr int kDitherTaps = R8BGPU_DITHER_MAX_TAPS;

// correctly rounded, never contracted into an FMA (the host side is built with -ffp-contract=off)
R8B_HD double dq_mul(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
R8B_HD double dq_add(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

// d for output n: SplitMix64's finaliser of seed + (n + 1) * golden gamma; the difference of two 32-bit uniforms scaled by
// 2^-32 is exact in double and triangular on (-1, 1)
R8B_HD double dither_tpdf(unsigned long long seed, long long n)
{
    unsigned long long z = seed + (unsigned long long) (n + 1) * 0x9E3779B97F4A7C15ull;
    z ^= z >> 30;
    z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27;
    z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return (double) (z >> 32) * (1.0 / 4294967296.0) - (double) (z & 0xFFFFFFFFull) * (1.0 / 4294967296.0);
}

// The integer range a format's values are saturated to: U8 stores an int8 value plus 128, and µ-law / A-law store the
// G.711 code of the int16 value (r8b_codec.cuh), so they quantise in the int16 domain.
R8B_HD void dither_range(int fmt, long long& lo, long long& hi)
{
    lo = -2147483647LL - 1, hi = 2147483647LL;
    if (fmt == FMT_U8) lo = -128, hi = 127;
    if (fmt == FMT_S16 || fmt == FMT_ULAW || fmt == FMT_ALAW) lo = -32768, hi = 32767;
    if (fmt == FMT_S24) lo = -8388608, hi = 8388607;
}

// One output: v = fl(y * scale) of output n; c[k-1] = c_k (k <= K), eh[k-1] = e[n-k] on entry, shifted by one with e[n]
// on return.  Returns the stored value.
R8B_HD long long dither_step(const double* c, int K, double* eh, unsigned long long seed, long long n, double v, long long lo,
                             long long hi)
{
    double s = 0.0;
#pragma unroll
    for (int k = kDitherTaps; k >= 1; k--)
        if (k <= K) s = dq_add(s, dq_mul(c[k - 1], eh[k - 1]));
    long long out;
    double e;
    if (!(fabs(v) <= DBL_MAX)) { // NaN -> 0, +-inf -> the limits: what the cast stores
        out = v != v ? 0 : (v > 0.0 ? hi : lo);
        e = 0.0;
    } else {
        const double w = dq_add(v, -s);
        const double q = rint(dq_add(w, dither_tpdf(seed, n)));
        e = dq_add(q, -w);
        out = q != q ? 0 : (q <= (double) lo ? lo : (q >= (double) hi ? hi : (long long) q));
    }
#pragma unroll
    for (int k = kDitherTaps - 1; k >= 1; k--) eh[k] = eh[k - 1];
    eh[0] = e;
    return out;
}

} // namespace r8bgpu

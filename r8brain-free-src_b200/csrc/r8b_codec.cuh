// r8b_codec.cuh -- the one-byte sample formats (include/r8bgpu.h, "caller-side sample formats"): unsigned 8-bit PCM and
// G.711 µ-law / A-law, in the convention of Sun's public-domain g711.c as CPython's audioop uses it (16-bit linear in and
// out; encoding looks at the top 14 (µ-law) / 13 (A-law) bits).  Integer arithmetic only -- the segment is a bit scan, no
// table in memory, since divergent indices into a table serialise -- and __host__ __device__, so the device conversions,
// the fused kernel's loads and stores and the host quantiser all produce the same bits from this one module.
#pragma once
#include "r8b_fft.cuh"
#include "r8b_kernels.h"

namespace r8bgpu {

R8B_HD bool is_byte_format(int fmt) { return fmt == FMT_U8 || fmt == FMT_ULAW || fmt == FMT_ALAW; }

// floor(log2(v)) for v >= 1
R8B_HD int codec_ilog2(unsigned v)
{
#ifdef __CUDA_ARCH__
    return 31 - __clz((int) v);
#else
    return 31 - __builtin_clz(v);
#endif
}

R8B_HD int ulaw_decode(unsigned char code)
{
    const int u = ~code & 0xff;
    const int t = (((u & 0x0f) << 3) + 0x84) << ((u & 0x70) >> 4);
    return (u & 0x80) ? 0x84 - t : t - 0x84;
}

R8B_HD int alaw_decode(unsigned char code)
{
    const int a = code ^ 0x55;
    const int seg = (a & 0x70) >> 4;
    int t = (a & 0x0f) << 4;
    t = seg == 0 ? t + 8 : (t + 0x108) << (seg - 1);
    return (a & 0x80) ? t : -t;
}

// s: a 16-bit value (-32768..32767)
R8B_HD unsigned char ulaw_encode(int s)
{
    int v = s >> 2; // 14 bits
    int mask = 0xff;
    if (v < 0) {
        v = -v;
        mask = 0x7f;
    }
    // g711.c clips the magnitude at 8159 and returns the top code once the biased value passes 0x1fff; 8158 + 33 = 0x1fff
    // already gives that code, so clipping there keeps the segment below 8
    v = (v > 8158 ? 8158 : v) + 33;
    const int seg = codec_ilog2((unsigned) v) - 5; // v >= 33: seg >= 0
    return (unsigned char) (((seg << 4) | ((v >> (seg + 1)) & 0x0f)) ^ mask);
}

R8B_HD unsigned char alaw_encode(int s)
{
    int v = s >> 3; // 13 bits
    int mask = 0xd5;
    if (v < 0) {
        v = -v - 1;
        mask = 0x55;
    }
    const int seg = v < 32 ? 0 : codec_ilog2((unsigned) v) - 4; // v <= 4095: seg <= 7
    return (unsigned char) (((seg << 4) | ((v >> (seg < 2 ? 1 : seg)) & 0x0f)) ^ mask);
}

// The linear value of a stored byte: U8 -> -128..127, µ-law / A-law -> the 16-bit expansion.
R8B_HD int byte_decode(int fmt, unsigned char code)
{
    if (fmt == FMT_U8) return (int) code - 128;
    return fmt == FMT_ULAW ? ulaw_decode(code) : alaw_decode(code);
}

// The stored byte of q: U8 takes an int8 value, µ-law / A-law an int16 value (both already saturated).
R8B_HD unsigned char byte_encode(int fmt, int q)
{
    if (fmt == FMT_U8) return (unsigned char) (q + 128);
    return fmt == FMT_ULAW ? ulaw_encode(q) : alaw_encode(q);
}

// What a sample of fmt holds for silence (0.0): 128 for U8, 0xFF for µ-law, 0xD5 for A-law, zero bytes otherwise.
R8B_HD unsigned char silence_byte(int fmt) { return is_byte_format(fmt) ? byte_encode(fmt, 0) : 0; }

} // namespace r8bgpu

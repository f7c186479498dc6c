// r8b_fused_common.cuh -- pieces shared by the two fused "2x BlockConvolver -> FracInterpolator" kernels
// (r8b_fused.cu: tile pairs, one CTA per pair; r8b_fused2.cu: persistent CTA, two half-CTA pipelines).
// Everything here is plain arithmetic on pointers, so it also compiles for the host: the CPU emulation of
// the v2 kernel (tests/cpp/fused2_emul.cu) runs these very functions thread by thread.
#pragma once
#include "r8b_codec.cuh"
#include "r8b_dither.cuh"
#include "r8b_fft.cuh"
#include "r8b_kernels.h"

namespace r8bgpu {

// (the typed paths are kept out of line: inlined into the fused kernel they cost the fp64 path ~3 % through code size and
// register pressure, and they are not the hot case)
#ifdef __CUDA_ARCH__
#define R8B_HD_COLD __host__ __device__ __noinline__
#else
#define R8B_HD_COLD inline
#endif

// One sample of a planar typed block, widened exactly ((double) of the stored value) and scaled with a correctly
// rounded multiply -- bit for bit what k_cvt_planar (r8b_format.cu) produces.
R8B_HD_COLD double typed_load(const void* base, long long idx, int fmt, double scale)
{
    double x;
    switch (fmt) {
    case FMT_F32: x = (double) R8B_LDG(reinterpret_cast<const float*>(base) + idx); break;
    case FMT_S16: x = (double) R8B_LDG(reinterpret_cast<const short*>(base) + idx); break;
    case FMT_S32: x = (double) R8B_LDG(reinterpret_cast<const int*>(base) + idx); break;
    case FMT_S24: {
        const unsigned char* p = reinterpret_cast<const unsigned char*>(base) + 3 * idx; // packed little-endian
        x = (double) ((int) R8B_LDG(p) | ((int) R8B_LDG(p + 1) << 8) | ((int) (signed char) R8B_LDG(p + 2) << 16));
        break;
    }
    case FMT_U8:
    case FMT_ULAW:
    case FMT_ALAW: x = (double) byte_decode(fmt, R8B_LDG(reinterpret_cast<const unsigned char*>(base) + idx)); break;
    default: x = R8B_LDG(reinterpret_cast<const double*>(base) + idx); break;
    }
#ifdef __CUDA_ARCH__
    return __dmul_rn(x, scale);
#else
    return x * scale;
#endif
}

// (T) (y * scale): float rounds to nearest, integers truncate toward zero and saturate, NaN -> 0 (r8b_format.cu); U8 stores
// the int8 value + 128, µ-law / A-law the G.711 code of the int16 value.
// dc != nullptr: integer outputs of channels set to TPDF are dithered instead (flat: the launch has no shaped channel);
// the element index idx = ch * stride + (n - dbase) gives the channel and its output index n, and the last 16 outputs of
// the call leave their errors in the channel's history.
R8B_HD_COLD void typed_store(void* base, long long idx, int fmt, double scale, double y, const DitherCall* dc, long long stride,
                             long long dbase, int ch0)
{
#ifdef __CUDA_ARCH__
    y = __dmul_rn(y, scale);
#else
    y = y * scale;
#endif
    if (fmt == FMT_F32) {
        reinterpret_cast<float*>(base)[idx] = (float) y;
        return;
    }
    long long lo, hi;
    dither_range(fmt, lo, hi);
    long long v = 0;
    if (y == y) v = y <= (double) lo ? lo : (y >= (double) hi ? hi : (long long) y); // C cast truncates toward zero
    if (dc != nullptr && fabs(y) <= DBL_MAX) {
        const long long ch = idx / stride, g = ch0 + ch;
        const DitherCfg& d = dc->cfg[g];
        if (d.kind != R8BGPU_DITHER_OFF) {
            const long long n = dbase + (idx - ch * stride);
            const double q = rint(dq_add(y, dither_tpdf(d.seed, n)));
            v = q <= (double) lo ? lo : (q >= (double) hi ? hi : (long long) q);
            const DitherRec& r = dc->rec[g];
            const long long f = n - r.n0;
            if (f >= r.n - kDitherTaps) dc->err[g * kDitherTaps + ((r.m0 + f) & (kDitherTaps - 1))] = dq_add(q, -y);
        }
    }
    if (fmt == FMT_S16) {
        reinterpret_cast<short*>(base)[idx] = (short) v;
    } else if (fmt == FMT_S32) {
        reinterpret_cast<int*>(base)[idx] = (int) v;
    } else if (is_byte_format(fmt)) {
        reinterpret_cast<unsigned char*>(base)[idx] = byte_encode(fmt, (int) v);
    } else {
        unsigned char* p = reinterpret_cast<unsigned char*>(base) + 3 * idx;
        p[0] = (unsigned char) (v & 0xff);
        p[1] = (unsigned char) ((v >> 8) & 0xff);
        p[2] = (unsigned char) ((v >> 16) & 0xff);
    }
}

R8B_HD double src_read_f(const SrcView& v, int ch, long long n)
{
    if (n >= v.avail) return 0.0;
    if (n >= v.cur_base) {
        if (v.cur_fmt != FMT_F64) return typed_load(v.cur, (long long) ch * v.cur_stride + (n - v.cur_base), v.cur_fmt, v.cur_scale);
        return R8B_LDG(v.cur + (long long) ch * v.cur_stride + (n - v.cur_base));
    }
    return R8B_LDG(v.ring + (long long) ch * v.ring_stride + (n & v.ring_mask));
}

R8B_HD void dst_write_f(const DstView& v, int ch, long long idx, double x)
{
    v.ptr[(long long) ch * v.stride + ((idx - v.base) & v.mask)] = x;
}

constexpr int FM = 4096;            // FFT length of the fused kernels
constexpr int FPL = fft_padded_len(FM);

R8B_HD int ylay(int i, int ysh) { return i + (i >> ysh); }

// Twiddles from shared memory, laid out [q][r] so that the 16 consecutive lanes of a half-warp read 16
// consecutive entries (the natural [r*q] indexing is an up-to-16-way bank conflict for even q):
//   tw2t[q*16 + r] = W_256^(r q)            (r, q < 16)  -- passes with NCUR = 256
//   tw1t[q*16 + r] = W_M^(r q)              (r, q < 16)
//   W_M^(R q), R = 16 r_hi + r_lo < 256  =  tw2t[q*16 + r_hi] * tw1t[q*16 + r_lo]   -- passes with NCUR = M
// (one extra complex multiply, <= ~1.5 ulp, instead of walking a 64 KB table through L1/L2).
R8B_HD double2 tw_pair(const double2* __restrict__ tw2t, const double2* __restrict__ tw1t, int r, int q)
{
    const double2 c = tw2t[q * 16 + (r >> 4)], f = tw1t[q * 16 + (r & 15)];
    return make_double2(fma(c.x, f.x, -c.y * f.y), fma(c.x, f.y, c.y * f.x));
}

// Twiddles of one radix-16 butterfly, W^(r q) for q = 1..15, from FOUR table reads (q = 1, 2, 4, 8) and eleven
// products W^(r (a+b)) = W^(r a) W^(r b).  The passes are bound by shared-memory wavefronts, not by the fp64 pipe,
// and a twiddle read costs as much as a data read.  A derived twiddle carries one to three extra roundings (q = 15);
// measured end to end (cfg 2 and 3, rms error against the reference, parity bar 4 eps): fifteen reads 2.53 eps, six
// reads + nine single products 2.55, this variant 2.58.  `ld(q)` fetches a table value; use(q, w) is called once per
// q, in the order (q, q + 8), so only w1, w2, w3, w4, w8 stay live.
R8B_HD double2 cprod(double2 a, double2 b) { return make_double2(fma(a.x, b.x, -a.y * b.y), fma(a.x, b.y, a.y * b.x)); }

template <typename Ld, typename Use>
R8B_HD void twiddles16(Ld ld, Use use)
{
    const double2 w8 = ld(8), w1 = ld(1), w2 = ld(2), w4 = ld(4);
    use(8, w8);
    use(1, w1);
    use(9, cprod(w1, w8));
    use(2, w2);
    use(10, cprod(w2, w8));
    const double2 w3 = cprod(w1, w2);
    use(3, w3);
    use(11, cprod(w3, w8));
    use(4, w4);
    use(12, cprod(w4, w8));
    const double2 w5 = cprod(w1, w4);
    use(5, w5);
    use(13, cprod(w5, w8));
    const double2 w6 = cprod(w2, w4);
    use(6, w6);
    use(14, cprod(w6, w8));
    const double2 w7 = cprod(w3, w4);
    use(7, w7);
    use(15, cprod(w7, w8));
}

// One radix-16 DIF pass over blocks of NCUR points in padded shared memory; butterfly g of M/16.
template <int NCUR>
R8B_HD void fwd_pass(double2* __restrict__ s, const double2* __restrict__ tw2_s, int g)
{
    constexpr int D = NCUR / 16;
    const int blk = g / D, r = g % D;
    const int base = blk * NCUR + r;
    double2 v[16];
#pragma unroll
    for (int j = 0; j < 16; j++) v[j] = s[fft_pad(base + j * D)];
    Network<16, +1>::run(v);
    s[fft_pad(base)] = v[0];
    if (D > 1) { // NCUR == 256: W_256^(r q), [q][r] layout
        twiddles16([&](int q) { return tw2_s[q * 16 + r]; },
                   [&](int q, double2 w) { s[fft_pad(base + q * D)] = cmul<+1>(v[bitrev<16>(q)], w); });
    } else {
#pragma unroll
        for (int q = 1; q < 16; q++) s[fft_pad(base + q * D)] = v[bitrev<16>(q)];
    }
}

template <int NCUR>
R8B_HD void inv_pass(double2* __restrict__ s, const double2* __restrict__ tw2_s, int g)
{
    constexpr int D = NCUR / 16;
    const int blk = g / D, r = g % D;
    const int base = blk * NCUR + r;
    double2 v[16];
    v[0] = s[fft_pad(base)];
    if (D > 1) {
        twiddles16([&](int q) { return tw2_s[q * 16 + r]; },
                   [&](int q, double2 w) { v[q] = cmul<-1>(s[fft_pad(base + q * D)], w); });
    } else {
#pragma unroll
        for (int q = 1; q < 16; q++) v[q] = s[fft_pad(base + q * D)];
    }
    Network<16, -1>::run(v);
#pragma unroll
    for (int j = 0; j < 16; j++) s[fft_pad(base + j * D)] = v[bitrev<16>(j)];
}

} // namespace r8bgpu

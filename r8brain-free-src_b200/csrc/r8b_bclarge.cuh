// r8b_bclarge.cuh -- per-thread steps of the large-tile overlap-save BlockConvolver (k_bcl_gather, k_bcl_conv,
// k_bcl_scatter in r8b_kernels.cu).
//
// Same operator as k_blockconv<M, UP = 1> (CDSPBlockConvolver.h:252-354 on top of CDSPRealFFT.h:98-385): two tiles
// (a, b) of one channel packed as z = x_a + i x_b, one M-point transform, Y = Z .* G, one inverse, y_a + i y_b.  For
// M = R0 * 4096 (R0 = 4, 8, 16) the tile does not fit one CTA's shared memory, so the transform is split along its
// outermost radix-R0 digit, the way the 8192-point transform of r8b_fft.cuh runs its leading radix-2 pass:
//
//   A (gather)  thread n1 < 4096:  v[j] = z[n1 + 4096 j], j < R0;  radix-R0 DIF butterfly;  output r times W_M^(r n1)
//               -> scratch sub-block r, element n1.  Sub-block r then holds the frequencies k = r + R0 k2.
//   B (conv)    one CTA per sub-block: fft_forward<4096>, multiply by G in slot order, fft_inverse<4096>, all in
//               shared memory (r8b_fft.cuh).  Slot of frequency k: (k % R0) * 4096 + slot_of<4096>(k / R0).
//   C (scatter) thread n1: the sub-blocks' element n1 times conj W_M^(r n1), radix-R0 inverse butterfly
//               -> y[n1 + 4096 j]; positions [lg, lg + adv) of both tiles go to the destination, every D-th.
//
// Reference-exact power-of-two decimation injects the Nyquist value at bin M/(2D) as k_blockconv does; that bin and
// its mirror M - M/(2D) are multiples of R0, i.e. bins 4096/(2D) and 4096 - 4096/(2D) of sub-block 0.
//
// Every function takes the thread's indices explicitly, so the same code runs on the host, one "thread" after
// another, in tests/cpp/bclarge_emul.cpp (kernel boundaries = loop boundaries).
#pragma once
#include "r8b_fft.cuh"
#include "r8b_kernels.h"

namespace r8bgpu {
namespace bcl {

constexpr int SUB = 4096;                         // points of every in-shared-memory transform
constexpr int SUB_PL = fft_padded_len(SUB);       // double2 of its padded shared-memory buffer
constexpr int ITEM_NT = 256;                      // threads per CTA of the gather / scatter kernels

__host__ __device__ __forceinline__ constexpr int slot_of_large(int k, int r0) { return (k % r0) * SUB + slot_of<SUB>(k / r0); }

// source sample n of the stage's input stream (k_blockconv's src_read)
R8B_HD double src_at(const SrcView& v, int ch, long long n)
{
    if (n >= v.avail) return 0.0;
    if (n >= v.cur_base) return R8B_LDG(v.cur + (long long) ch * v.cur_stride + (n - v.cur_base));
    return R8B_LDG(v.ring + (long long) ch * v.ring_stride + (n & v.ring_mask));
}

// sample u of the tile stream: the source itself, or its zero-stuffed view (src_up > 1)
R8B_HD double tile_at(const BlockConvParams& p, const SrcView& v, int ch, long long u)
{
    if (p.src_up <= 1) return src_at(v, ch, u);
    return (u >= 0 && u % p.src_up == 0) ? src_at(v, ch, u / p.src_up) : 0.0;
}

R8B_HD void dst_put(const DstView& v, int ch, long long idx, double x)
{
    v.ptr[(long long) ch * v.stride + ((idx - v.base) & v.mask)] = x;
}

// One tile pair of one channel; unit = channel (of the launch group) * pairs + pair.
struct Pair {
    int ch;
    bool has_b;
    long long ma, mb; // first owned input-rate position of tiles a and b
};

R8B_HD int n_pairs(const BlockConvParams& p) { return (p.n_tiles + 1) >> 1; }

R8B_HD Pair pair_of(const BlockConvParams& p, int unit)
{
    Pair t;
    const int np = n_pairs(p);
    t.ch = unit / np;
    const int ta = 2 * (unit - t.ch * np);
    t.has_b = (ta + 1) < p.n_tiles;
    t.ma = p.m0 + (long long) ta * p.adv;
    t.mb = t.ma + p.adv;
    return t;
}

// A: thread n1 of a pair -- gather R0 samples of each tile at stride 4096, leading radix-R0 DIF pass, twiddle, store.
template <int R0>
R8B_HD void gather_item(const BcLargeParams& p, const SrcView& src, const Pair& t, int n1, double2* __restrict__ blk)
{
    const long long wa = t.ma - p.bc.lg + n1, wb = t.mb - p.bc.lg + n1;
    double2 v[R0];
#pragma unroll
    for (int j = 0; j < R0; j++) {
        const double xa = tile_at(p.bc, src, t.ch, wa + (long long) SUB * j);
        const double xb = t.has_b ? tile_at(p.bc, src, t.ch, wb + (long long) SUB * j) : 0.0;
        v[j] = make_double2(xa, xb);
    }
    Network<R0, +1>::run(v);
#pragma unroll
    for (int q = 0; q < R0; q++) {
        double2 x = v[bitrev<R0>(q)];
        if (q > 0) x = cmul<+1>(x, R8B_LDG(&p.tw_m[q * n1]));
        blk[q * SUB + n1] = x;
    }
}

// B, block-exact stages, sub-block 0 only (one thread): the reference's Nyquist term from the forward spectrum
R8B_HD double2 conv_nyquist(const BcLargeParams& p, const double2* zbuf)
{
    const int kq = SUB / (2 * p.bc.trunc);
    const double2 z1 = zbuf[fft_pad(slot_of<SUB>(kq))];
    const double2 z2 = zbuf[fft_pad(slot_of<SUB>(SUB - kq))];
    const double2 xa = make_double2(0.5 * (z1.x + z2.x), 0.5 * (z1.y - z2.y));
    const double2 xb = make_double2(0.5 * (z1.y + z2.y), 0.5 * (z2.x - z1.x));
    return make_double2(p.bc.nyq_gain * (xa.x - xa.y), p.bc.nyq_gain * (xb.x - xb.y));
}

// B: slot s of sub-block r -- multiply by the filter spectrum (or put the Nyquist term in its bin)
R8B_HD void conv_mul_item(const BcLargeParams& p, double2* zbuf, int r, int s, bool nyq_here, double2 nyq)
{
    const double2 z = zbuf[fft_pad(s)];
    const double2 g = R8B_LDG(&p.bc.spec[r * SUB + s]);
    zbuf[fft_pad(s)] = (nyq_here && s == slot_of<SUB>(SUB / (2 * p.bc.trunc))) ? nyq : cmul<+1>(z, g);
}

// C: thread n1 of a pair -- twiddle, trailing radix-R0 inverse pass, owned positions of both tiles to the destination.
template <int R0>
R8B_HD void scatter_item(const BcLargeParams& p, const DstView& dst, const Pair& t, int n1, const double2* __restrict__ blk)
{
    double2 v[R0];
#pragma unroll
    for (int q = 0; q < R0; q++) {
        double2 x = blk[q * SUB + n1];
        if (q > 0) x = cmul<-1>(x, R8B_LDG(&p.tw_m[q * n1]));
        v[q] = x;
    }
    Network<R0, -1>::run(v);
    const BlockConvParams& b = p.bc;
    const long long t_lo = b.e0 * b.down, t_hi = b.e1 * b.down; // y indices [t_lo, t_hi) are wanted
    const long long cnt_a = b.m1 - t.ma < b.adv ? b.m1 - t.ma : b.adv;
    const long long cnt_b = !t.has_b ? 0 : b.m1 - t.mb < b.adv ? b.m1 - t.mb : b.adv;
#pragma unroll
    for (int j = 0; j < R0; j++) {
        const double2 y = v[bitrev<R0>(j)];
        const long long i = (long long) n1 + (long long) SUB * j - b.lg; // owned local index of both tiles
        if (i < 0) continue;
        if (i < cnt_a) {
            const long long tt = t.ma + i;
            if (tt >= t_lo && tt < t_hi && (b.down == 1 || tt % b.down == 0)) dst_put(dst, t.ch, tt / b.down, y.x);
        }
        if (i < cnt_b) {
            const long long tt = t.mb + i;
            if (tt >= t_lo && tt < t_hi && (b.down == 1 || tt % b.down == 0)) dst_put(dst, t.ch, tt / b.down, y.y);
        }
    }
}

} // namespace bcl
} // namespace r8bgpu

// r8b_fused2_core.cuh -- per-thread phase functions of the v2 fused kernel (r8b_fused2.cu).
//
// Same operator as r8b_fused.cu -- 2x BlockConvolver (CDSPBlockConvolver.h:252-354 on top of
// CDSPRealFFT.h:98-385) followed by the whole-stepping fractional interpolator
// (CDSPFracInterpolator.h:991-1060) -- but one TILE per 256-thread half-CTA instead of one tile PAIR per
// 512-thread CTA, so that two tiles in different phases share an SM:
//
//   forward : real input x[w .. w+4096)  ->  z[m] = x[2m] + i x[2m+1]  ->  2048-point complex DIF FFT
//             (radix 8 from registers, then radix 16, 16; spectrum in slot order)
//   C       : X[k] = E[k] + W_M^k O[k] from (Z[k], Z[N-k]);  Y = X * G on all 4096 bins (X Hermitian),
//             G = FFT(g_0 + i g_1)/(2M) the polyphase-packed low-pass (same table as v1)
//   inverse : 4096-point complex, radix 16 x 3; element e of the result = y[2(w+e)] + i y[2(w+e)+1]
//   interp  : out[j] = sum_i bank[phase(j)][i] * y[p_j - fll + i] out of shared memory
//
// Every function takes the thread's index explicitly and touches only its arguments, so the same code
// runs on the host, one "thread" after another, in tests/cpp/fused2_emul.cu (barriers = loop boundaries).
#pragma once
#include <climits>

#include "r8b_fused_common.cuh"
#include "r8b_poly.cuh"

namespace r8bgpu {
namespace f2 {

constexpr int FN = 2048;   // complex length of the forward transform (real length FM = 4096)
constexpr int FPL2 = FPL + 16; // double2 per tile buffer: room for the skewed copy of the forward result in its upper half
constexpr int SKEW0 = fft_padded_len(FN); // where that copy starts (= where a bulk-copied input tile lands)
constexpr int HT = 256;    // threads of one half-CTA pipeline
constexpr int IQ2 = 3;     // stepping cycles per lane in the interpolation register tile

struct Tile {
    int ch;
    long long A0, A1;      // owned 2x-rate positions [A0, A1)
    long long w;           // input index of local sample 0 of the FFT window
};

R8B_HD Tile tile_of(const FusedParams& p, int u)
{
    Tile t;
    t.ch = u / p.n_tiles;
    const int ti = u - t.ch * p.n_tiles;
    t.A0 = p.p_lo + (long long) ti * p.span;
    t.A1 = t.A0 + p.span;
    if (t.A1 > p.p_hi) t.A1 = p.p_hi;
    // valid y of the tile starts at A0 - yl (even) = 2 * (first valid m) [up 2; up 1: = first valid m]; the window starts lg earlier
    t.w = (p.up == 1 ? t.A0 - p.yl : (t.A0 - p.yl) / 2) - p.lg;
    return t;
}

// Where the tile's 4096 input samples are contiguous in memory: the caller's block (first stage of a chain), or the
// source ring when the window neither wraps nor reaches past the samples written so far (later stages).
R8B_HD const double* tile_run(const SrcView& src, const Tile& t)
{
    if (t.w >= src.cur_base && t.w + FM <= src.avail)
        return src.cur_fmt == FMT_F64 ? src.cur + (long long) t.ch * src.cur_stride + (t.w - src.cur_base) : nullptr;
    if (t.w >= 0 && t.w + FM <= src.avail && t.w + FM <= src.cur_base) {
        const long long i0 = t.w & src.ring_mask;
        if (i0 + FM <= src.ring_mask + 1) return src.ring + (long long) t.ch * src.ring_stride + i0;
    }
    return nullptr;
}

// Which way the samples arrive: 0 = every sample individually (history ring across a wrap, before the start, or past
// the available input), 1 = plain loads from a contiguous run, 2 = one bulk copy (16-byte aligned run), 3 = a run of
// the caller's block in a narrower sample format, widened while it is gathered.
R8B_HD int tile_input_path(const SrcView& src, const Tile& t)
{
    if (src.cur_fmt != FMT_F64 && t.w >= src.cur_base && t.w + FM <= src.avail) return 3;
    const double* a = tile_run(src, t);
    if (a == nullptr) return 0;
    return (reinterpret_cast<unsigned long long>(a) & 15) == 0 ? 2 : 1;
}

// z[m], m = r + 256 j, straight from global memory (paths 0 and 1)
R8B_HD void gather_tile(double2 (&v)[8], const SrcView& src, const Tile& t, int path, int r)
{
    if (path == 3) {
        const long long i0 = (long long) t.ch * src.cur_stride + (t.w - src.cur_base) + 2 * r;
#pragma unroll
        for (int j = 0; j < 8; j++)
            v[j] = make_double2(typed_load(src.cur, i0 + 512 * j, src.cur_fmt, src.cur_scale),
                                typed_load(src.cur, i0 + 512 * j + 1, src.cur_fmt, src.cur_scale));
    } else if (path != 0) {
        const double* __restrict__ a = tile_run(src, t) + 2 * r;
        if ((reinterpret_cast<unsigned long long>(a) & 15) == 0) {
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = R8B_LDG(reinterpret_cast<const double2*>(a + 512 * j));
        } else {
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = make_double2(R8B_LDG(a + 512 * j), R8B_LDG(a + 512 * j + 1));
        }
    } else {
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const long long n = t.w + 2 * (r + 256 * j);
            v[j] = make_double2(src_read_f(src, t.ch, n), src_read_f(src, t.ch, n + 1));
        }
    }
}

// forward pass 1: radix 8 on registers, NCUR = FN, D = 256; twiddle W_2048^(r q) = W_4096^(r 2q): q = 1, 2, 4 from the tables,
// the other four as products (see twiddles16)
R8B_HD void fwd_pass1_r8(double2 (&v)[8], double2* __restrict__ s, const double2* __restrict__ twc,
                         const double2* __restrict__ twf, int r)
{
    Network<8, +1>::run(v);
    const double2 w1 = tw_pair(twc, twf, r, 2), w2 = tw_pair(twc, twf, r, 4), w4 = tw_pair(twc, twf, r, 8);
    const double2 w3 = cprod(w1, w2);
    s[fft_pad(r)] = v[0];
    s[fft_pad(r + 1 * 256)] = cmul<+1>(v[bitrev<8>(1)], w1);
    s[fft_pad(r + 2 * 256)] = cmul<+1>(v[bitrev<8>(2)], w2);
    s[fft_pad(r + 3 * 256)] = cmul<+1>(v[bitrev<8>(3)], w3);
    s[fft_pad(r + 4 * 256)] = cmul<+1>(v[bitrev<8>(4)], w4);
    s[fft_pad(r + 5 * 256)] = cmul<+1>(v[bitrev<8>(5)], cprod(w1, w4));
    s[fft_pad(r + 6 * 256)] = cmul<+1>(v[bitrev<8>(6)], cprod(w2, w4));
    s[fft_pad(r + 7 * 256)] = cmul<+1>(v[bitrev<8>(7)], cprod(w3, w4));
}

// C (up-factor 1; the 2x pair fuses this phase into its first inverse pass, see cd1_*), first half: this thread's four
// frequency pairs (k, N-k), k <= N/2.  In slot order (k = q1 + 8 q2 + 128 q3,
// slot = 256 q1 + 16 q2 + q3) those are the slots with q3 < 8; a thread takes runs of 8 consecutive slots.
R8B_HD int c_freq(int ht, int u) { return freq_of<FN>(16 * ((ht >> 3) + 32 * u) + (ht & 7)); }

R8B_HD void c_load(const double2* __restrict__ buf, int ht, double2 (&z1)[4], double2 (&z2)[4])
{
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int s1 = 16 * ((ht >> 3) + 32 * u) + (ht & 7);
        const int k = freq_of<FN>(s1);
        const int s2 = slot_of<FN>((FN - k) & (FN - 1));
        z1[u] = buf[fft_pad(s1)];
        z2[u] = buf[fft_pad(s2)];
    }
}

// ---- phase C fused into the first inverse pass (up-factor 2) -------------------------------------------------------
// The first inverse pass gives butterfly g = 16 q1 + q2 the sixteen bins k = q1 + 16 q2 + 256 q3 (slots 16 g + q3).  They
// are X[kappa_t] G and X[kappa_t + N] G for kappa_t = q1 + 16 q2 + 256 t, t < 8, and both come from the forward values
// Z[kappa_t], Z[N - kappa_t]: a thread that fetches those sixteen values computes its own butterfly inputs, and the
// separate split pass -- its stores, the butterfly's loads, one barrier -- disappears.  For the fetches to stay
// conflict-free the last forward pass leaves Z in a SKEWED layout in the buffer's upper half,
//     skew(slot) = slot + slot/16 + slot/128
// (a quarter-warp reads blocks B0 + 2i, i < 8: the extra slot/128 term separates the two groups of four that the plain
// slot/16 padding puts on the same banks).  W_M^kappa_t = W_M^(q1 + 16 q2) * W_16^t: one table value per thread and the
// constant roots of the radix-16 network.  Operands in thread order (FusedParams::cd_tab): [q3 < 16][g < 256] spectrum,
// then [g < 256] twiddles.
R8B_HD int skew(int slot) { return slot + (slot >> 4) + (slot >> 7); }

// last forward pass (16-point blocks), out of place into the skewed layout
R8B_HD void fwd_pass16_skew(double2* __restrict__ buf, int g)
{
    double2 v[16];
#pragma unroll
    for (int j = 0; j < 16; j++) v[j] = buf[fft_pad(16 * g + j)];
    Network<16, +1>::run(v);
#pragma unroll
    for (int q = 0; q < 16; q++) buf[SKEW0 + skew(16 * g + q)] = v[bitrev<16>(q)];
}

R8B_HD void cd1_load(const double2* __restrict__ buf, int g, double2 (&z1)[8], double2 (&z2)[8])
{
    const int k0 = (g >> 4) + 16 * (g & 15);
#pragma unroll
    for (int t = 0; t < 8; t++) {
        const int k = k0 + 256 * t;
        z1[t] = buf[SKEW0 + skew(slot_of<FN>(k))];
        z2[t] = buf[SKEW0 + skew(slot_of<FN>((FN - k) & (FN - 1)))];
    }
}

template <int T>
R8B_HD void cd1_bin(const FusedParams& p, int g, double2 w0, double2 z1, double2 z2, double2 (&v)[16])
{
    const double2 a = make_double2(z1.x + z2.x, z1.y - z2.y);
    const double2 b = make_double2(z1.y + z2.y, z2.x - z1.x);
    const double2 wb = cmul<+1>(b, mul_root<16, T, +1>(w0));
    const double2 x0 = make_double2(a.x + wb.x, a.y + wb.y);
    const double2 x1 = make_double2(a.x - wb.x, a.y - wb.y);
    v[T] = cmul<+1>(x0, R8B_LDG(&p.cd_tab[T * HT + g]));
    v[T + 8] = cmul<+1>(x1, R8B_LDG(&p.cd_tab[(T + 8) * HT + g]));
}

// butterfly g of the first inverse pass, inputs computed from the forward values
R8B_HD void cd1_compute(const FusedParams& p, double2* __restrict__ buf, int g, const double2 (&z1)[8], const double2 (&z2)[8])
{
    const double2 w0 = R8B_LDG(&p.cd_tab[16 * HT + g]);
    double2 v[16];
    cd1_bin<0>(p, g, w0, z1[0], z2[0], v);
    cd1_bin<1>(p, g, w0, z1[1], z2[1], v);
    cd1_bin<2>(p, g, w0, z1[2], z2[2], v);
    cd1_bin<3>(p, g, w0, z1[3], z2[3], v);
    cd1_bin<4>(p, g, w0, z1[4], z2[4], v);
    cd1_bin<5>(p, g, w0, z1[5], z2[5], v);
    cd1_bin<6>(p, g, w0, z1[6], z2[6], v);
    cd1_bin<7>(p, g, w0, z1[7], z2[7], v);
    Network<16, -1>::run(v);
#pragma unroll
    for (int j = 0; j < 16; j++) buf[fft_pad(16 * g + j)] = v[bitrev<16>(j)];
}

// ---- the same, with the filter spectrum in its symmetric half-size form (FusedParams::cs_tab, in shared memory) ------
// The low-pass is zero-phase (h[-n] = h[n]), so with g0[j] = h[2j] and g1[j] = h[2j+1] = g1[-1-j]:  FFT(g0) = A0 is real
// and even, and FFT(g1)[k] = A1[k] phi(k) with the half-bin phase phi(k) = e^(+i pi k / M) and A1 real, A1[M-k] = -A1[k].
// With a0 = A0/(2M), a1 = A1/(2M), the two bins a butterfly needs for each t < 8 are
//     G[kappa]     = a0[kappa] + i a1[kappa] phi(kappa)
//     G[kappa + N] = a0[N - kappa] + a1[N - kappa] phi(kappa)
// so the pairs (a0[k], a1[k]), k = 0..N (2049 x 16 bytes), stand for all 4096 bins, and one phase serves both bins:
// phi(kappa_t) = phi_g rho^t with phi_g = phi(q1 + 16 q2) per thread and rho = e^(i pi / 16).  Pair k sits at
// cs_entry(k): thread order [t][g] for k = q1 + 16 q2 + 256 t, k = N last.  A thread's second read,
// cs_entry(N - kappa_t) = cs_entry(N - kappa_0) - 256 t, lands for a warp on two adjacent runs of 16 entries (512
// contiguous bytes), like its first.  After the N + 1 pairs: [g < 256] W_M^kappa_0, then [g < 256] phi_g.
constexpr int CS_PAIRS = FN + 1;
R8B_HD int cs_entry(int k) { return (k & ~255) | ((k & 15) << 4) | ((k >> 4) & 15); }
R8B_HD int cs_second(int g) { return cs_entry(FN - ((g >> 4) + 16 * (g & 15))); }

// a * e^(i pi T / 16), T < 8 (compile-time)
template <int T>
R8B_HD double2 rot32(double2 a)
{
    if constexpr ((T & 1) == 0) {
        return mul_root<16, T / 2, -1>(a);
    } else {
        constexpr double c1 = 0.98078528040323044913, s1 = 0.19509032201612826785; // cos, sin (pi/16)
        constexpr double c3 = 0.83146961230254523708, s3 = 0.55557023301960222474; // cos, sin (3 pi/16)
        constexpr double c = T == 1 ? c1 : T == 3 ? c3 : T == 5 ? s3 : s1;
        constexpr double s = T == 1 ? s1 : T == 3 ? s3 : T == 5 ? c3 : c1;
        return make_double2(fma(a.x, c, -a.y * s), fma(a.x, s, a.y * c));
    }
}

// G[kappa] from the pair at kappa, G[kappa + N] from the pair at N - kappa (ph = phi(kappa))
R8B_HD double2 cs_bin_lo(double2 e, double2 ph) { return make_double2(fma(-e.y, ph.y, e.x), e.y * ph.x); }
R8B_HD double2 cs_bin_hi(double2 f, double2 ph) { return make_double2(fma(f.y, ph.x, f.x), f.y * ph.y); }

template <int T>
R8B_HD void cd1s_bin(const double2* __restrict__ cs, int i1, int i2, double2 w0, double2 phg, double2 z1, double2 z2,
                     double2 (&v)[16])
{
    const double2 a = make_double2(z1.x + z2.x, z1.y - z2.y);
    const double2 b = make_double2(z1.y + z2.y, z2.x - z1.x);
    const double2 wb = cmul<+1>(b, mul_root<16, T, +1>(w0));
    const double2 x0 = make_double2(a.x + wb.x, a.y + wb.y);
    const double2 x1 = make_double2(a.x - wb.x, a.y - wb.y);
    const double2 ph = rot32<T>(phg);
    v[T] = cmul<+1>(x0, cs_bin_lo(cs[i1 + 256 * T], ph));
    v[T + 8] = cmul<+1>(x1, cs_bin_hi(cs[i2 - 256 * T], ph));
}

// cd1_compute with the spectrum pairs at cs (shared memory); w0 = W_M^kappa_0 and phg = phi_g of butterfly g
R8B_HD void cd1s_compute(const double2* __restrict__ cs, double2 w0, double2 phg, double2* __restrict__ buf, int g,
                         const double2 (&z1)[8], const double2 (&z2)[8])
{
    const int i1 = g, i2 = cs_second(g); // entries of (t = 0, kappa) and (t = 0, N - kappa)
    double2 v[16];
    cd1s_bin<0>(cs, i1, i2, w0, phg, z1[0], z2[0], v);
    cd1s_bin<1>(cs, i1, i2, w0, phg, z1[1], z2[1], v);
    cd1s_bin<2>(cs, i1, i2, w0, phg, z1[2], z2[2], v);
    cd1s_bin<3>(cs, i1, i2, w0, phg, z1[3], z2[3], v);
    cd1s_bin<4>(cs, i1, i2, w0, phg, z1[4], z2[4], v);
    cd1s_bin<5>(cs, i1, i2, w0, phg, z1[5], z2[5], v);
    cd1s_bin<6>(cs, i1, i2, w0, phg, z1[6], z2[6], v);
    cd1s_bin<7>(cs, i1, i2, w0, phg, z1[7], z2[7], v);
    Network<16, -1>::run(v);
#pragma unroll
    for (int j = 0; j < 16; j++) buf[fft_pad(16 * g + j)] = v[bitrev<16>(j)];
}

// inverse, last pass (NCUR = M, D = 256): loads + butterfly; the results leave through y_store()
R8B_HD void inv3_load(const double2* __restrict__ buf, const double2* __restrict__ twc, const double2* __restrict__ twf,
                      int g, double2 (&v)[16])
{
    v[0] = buf[fft_pad(g)];
    twiddles16([&](int q) { return tw_pair(twc, twf, g, q); },
               [&](int q, double2 w) { v[q] = cmul<-1>(buf[fft_pad(g + q * 256)], w); });
    Network<16, -1>::run(v);
}

template <bool PADV>
R8B_HD void y_store(double2* __restrict__ buf, const double2 (&v)[16], int g, long long w, int ysh)
{
    double* yb = reinterpret_cast<double*>(buf);
    if (w < 0) { // only the first tile of a stream reaches before sample 0 (tile-uniform branch)
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int e = g + j * 256;              // local input-rate position
            double2 x = v[bitrev<16>(j)];
            if (w + e < 0) x = make_double2(0.0, 0.0); // the reference's interpolator starts from silence
            if (!PADV) {
                reinterpret_cast<double2*>(yb)[e] = x;
            } else {
                yb[ylay(2 * e, ysh)] = x.x;
                yb[ylay(2 * e + 1, ysh)] = x.y;
            }
        }
        return;
    }
#pragma unroll
    for (int j = 0; j < 16; j++) {
        const int e = g + j * 256;
        const double2 x = v[bitrev<16>(j)];
        if (!PADV) {
            reinterpret_cast<double2*>(yb)[e] = x;
        } else {
            yb[ylay(2 * e, ysh)] = x.x;
            yb[ylay(2 * e + 1, ysh)] = x.y;
        }
    }
}

// ---- up-factor 1 (BlockConvolver 1/1 -> interpolator: the tail of every decimating chain) -------------------------
// The tile's 4096 real outputs come from a 2048-point complex INVERSE transform, the mirror of the real-input forward
// one:  with Y[k] = X[k] H[k] (k = 0..N, Hermitian beyond),  Z'[k] = (Y[k] + conj Y[N-k]) + i W_M^-k (Y[k] - conj Y[N-k])
// and IFFT_N(Z')[m] = y[2m] + i y[2m+1].  Per pair (k, N-k), from the forward values z1 = Z[k], z2 = Z[N-k]:
//   x0 = 2X[k] = a + W^k b,  x1 = 2X[k+N] = a - W^k b   (a = Z[k] + conj Z[N-k] = 2E[k], b = -i (Z[k] - conj Z[N-k]) = 2O[k]);   2X[N-k] = conj x1
//   p = x0 h0,  q = conj(x1) h1          (h0 = H[k]/2, h1 = H[N-k]/2; H = FFT(h)/M is real up to rounding)
//   s = p + conj q,  t = i conj(W^k) (p - conj q);   Z'[k] = s + t,  Z'[N-k] = conj(s - t)
// k = 0 pairs DC with the Nyquist bin (h1 = H[N]/2) and k = N/2 pairs with itself: both write one slot.
R8B_HD void c1_pair_ops(double2* __restrict__ buf, int k, double2 z1, double2 z2, double2 w, double2 h0, double2 h1)
{
    const double2 a = make_double2(z1.x + z2.x, z1.y - z2.y);
    const double2 b = make_double2(z1.y + z2.y, z2.x - z1.x);
    const double2 wb = cmul<+1>(b, w);
    const double2 x0 = make_double2(a.x + wb.x, a.y + wb.y);
    const double2 x1c = make_double2(a.x - wb.x, wb.y - a.y); // conj(a - wb)
    const double2 pp = cmul<+1>(x0, h0), qq = cmul<+1>(x1c, h1);
    const double2 sm = make_double2(pp.x + qq.x, pp.y - qq.y);
    const double2 df = make_double2(pp.x - qq.x, pp.y + qq.y);
    const double2 cd = cmul<-1>(df, w);                        // conj(W^k) (p - conj q)
    const double2 tt = make_double2(-cd.y, cd.x);              // times i
    const int s0 = slot_of<FN>(k), s1 = slot_of<FN>((FN - k) & (FN - 1));
    buf[fft_pad(s0)] = make_double2(sm.x + tt.x, sm.y + tt.y);
    if (s1 != s0) buf[fft_pad(s1)] = make_double2(sm.x - tt.x, tt.y - sm.y);
}

R8B_HD void c1_pair_tab(const FusedParams& p, double2* __restrict__ buf, int ht, int u, double2 z1, double2 z2)
{
    const double2* __restrict__ ct = p.c_tab + (u * 3) * HT + ht;
    c1_pair_ops(buf, c_freq(ht, u), z1, z2, R8B_LDG(ct), R8B_LDG(ct + HT), R8B_LDG(ct + 2 * HT));
}

R8B_HD void c1_pair_mid(const FusedParams& p, double2* __restrict__ buf, double2 ze)
{
    const double2* __restrict__ ct = p.c_tab + 12 * HT;
    c1_pair_ops(buf, FN / 2, ze, ze, R8B_LDG(ct), R8B_LDG(ct + 1), R8B_LDG(ct + 2));
}

// inverse, last pass of the 2048-point transform (radix 8, D = 256): mirror of fwd_pass1_r8
R8B_HD void inv1_last_load(const double2* __restrict__ buf, const double2* __restrict__ twc, const double2* __restrict__ twf, int r,
                           double2 (&v)[8])
{
    const double2 w1 = tw_pair(twc, twf, r, 2), w2 = tw_pair(twc, twf, r, 4), w4 = tw_pair(twc, twf, r, 8);
    const double2 w3 = cprod(w1, w2);
    v[0] = buf[fft_pad(r)];
    v[1] = cmul<-1>(buf[fft_pad(r + 1 * 256)], w1);
    v[2] = cmul<-1>(buf[fft_pad(r + 2 * 256)], w2);
    v[3] = cmul<-1>(buf[fft_pad(r + 3 * 256)], w3);
    v[4] = cmul<-1>(buf[fft_pad(r + 4 * 256)], w4);
    v[5] = cmul<-1>(buf[fft_pad(r + 5 * 256)], cprod(w1, w4));
    v[6] = cmul<-1>(buf[fft_pad(r + 6 * 256)], cprod(w2, w4));
    v[7] = cmul<-1>(buf[fft_pad(r + 7 * 256)], cprod(w3, w4));
    Network<8, -1>::run(v);
}

// element m = r + 256 j of the result is y[2m] + i y[2m+1], local positions of the 1x stream (position w + index)
template <bool PADV>
R8B_HD void y_store1(double2* __restrict__ buf, const double2 (&v)[8], int r, long long w, int ysh)
{
    double* yb = reinterpret_cast<double*>(buf);
    const bool head = w < 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int m = r + j * 256;
        double2 x = v[bitrev<8>(j)];
        if (head) { // the reference's interpolator starts from silence
            if (w + 2 * m < 0) x.x = 0.0;
            if (w + 2 * m + 1 < 0) x.y = 0.0;
        }
        if (!PADV) {
            reinterpret_cast<double2*>(yb)[m] = x;
        } else {
            yb[ylay(2 * m, ysh)] = x.x;
            yb[ylay(2 * m + 1, ysh)] = x.y;
        }
    }
}

// Tile-level bookkeeping of the interpolation: everything the per-task code needs afterwards is 32-bit and relative to
// the tile.  Returns the tile's first output index ja.
//   s_i[0] outputs of the tile, [1] last (shifted) stepping cycle, [2] output index of (cycle 0, phase 0)
//   relative to the tile's first output, [3] y index of the window of (cycle 0, offset 0)
R8B_HD long long interp_tile(const FusedParams& p, const Tile& t, int* s_i)
{
    long long ja = (t.A0 * p.out_step + p.in_step - 1) / p.in_step;
    long long jb = (t.A1 * p.out_step + p.in_step - 1) / p.in_step;
    if (ja < p.e0) ja = p.e0;
    if (jb > p.e1) jb = p.e1;
    const long long ad = ja - p.delta, bd = jb - 1 - p.delta;
    const long long c_first = ad >= 0 ? ad / p.out_step : -1, c_last = bd >= 0 ? bd / p.out_step : -1;
    s_i[0] = jb > ja ? (int) (jb - ja) : 0;
    s_i[1] = (int) (c_last - c_first);
    s_i[2] = (int) (c_first * p.out_step - ja);
    s_i[3] = (int) (c_first * p.in_step - p.fll - (p.up == 1 ? 1 : 2) * t.w);
    return ja;
}

// The same for one tile of one channel, with where its outputs go: s_i[0..3] as above, *s_op = the slot of the tile's
// first output, s_i[4..5] = its element index in a typed linear destination (low, high word).
R8B_HD void interp_prepare(const FusedParams& p, const DstView& dst, const Tile& t, int* s_i, double** s_op)
{
    const long long ja = interp_tile(p, t, s_i);
    *s_op = dst.ptr + (long long) t.ch * dst.stride + ((ja - dst.base) & dst.mask);
    const long long e0 = (long long) t.ch * dst.stride + (ja - dst.base); // typed destinations: element index, [4..5]
    s_i[4] = (int) (e0 & 0xffffffffLL);
    s_i[5] = (int) (e0 >> 32);
}

// ---- the call's tile table --------------------------------------------------------------------------------------
// A tile's bookkeeping depends on its index ti within the call alone (A0 = p_lo + ti span; channels differ only by their
// destination row, ch * stride), and it costs 64-bit divisions.  So the kernel computes it once per tile index in its
// prologue, one thread per entry, into shared memory (FusedParams::n_tab entries at byte offset tab_off), and every
// tile of every channel reads its entry there.  A tile whose index is past n_tab -- a call with more tiles than the
// shared memory the plan leaves over holds -- computes its own entry (thread 255 of its half, during phase A).
struct TileEntry {
    int s[4];      // interp_tile's s_i[0..3]; order-2 bank (mode 1): s[0], s[1] = first output of the call at or past A0, A1
    long long off; // ja - dst.base: the tile's first output is element ch * stride + off of a linear destination, slot
                   // (off & mask) of row ch of a ring
};

R8B_HD TileEntry tile_entry(const FusedParams& p, long long dst_base, int ti)
{
    const Tile t = tile_of(p, ti); // (channel 0)
    TileEntry e;
    if (p.mode == 1) {
        const long long nk = p.e1 - p.e0;
        e.s[0] = (int) poly_first_k(p, t.A0, nk);
        e.s[1] = (int) poly_first_k(p, t.A1, nk);
        e.s[2] = e.s[3] = 0;
        e.off = 0;
    } else {
        e.off = interp_tile(p, t, e.s) - dst_base;
    }
    return e;
}

// Lane geometry of the interpolation: a warp covers CL = 32 >> GLOG stepping cycles x GL = 1 << GLOG phase
// groups per instruction; a lane owns IR consecutive phases of its group in IQ2 cycles (CL apart).
template <int IR, int GLOG>
struct TaskGeom {
    static constexpr int GL = 1 << GLOG, CL = 32 >> GLOG, CYC = CL * IQ2;
    int grp, r0, o0, cb;   // phase group (clamped), its first phase, its window offset, first cycle of the lane
    bool gvalid;
    R8B_HD void set(const FusedParams& p, const int* __restrict__ s_goff, int task, int lane)
    {
        const int n_groups = (p.out_step + IR - 1) / IR;
        const int n_gt = (n_groups + GL - 1) / GL;
        const int gt = task % n_gt, chunk = task / n_gt;
        grp = gt * GL + (lane >> (5 - GLOG));
        gvalid = grp < n_groups;
        if (!gvalid) grp = n_groups - 1;
        r0 = p.delta + grp * IR;
        o0 = s_goff[grp];
        cb = chunk * CYC + (lane & (CL - 1));
    }
    static R8B_HD int n_tasks(const FusedParams& p, int c_cnt)
    {
        const int n_groups = (p.out_step + IR - 1) / IR;
        return ((n_groups + GL - 1) / GL) * ((c_cnt + CYC) / CYC);
    }
};

// y indices of the lane's IQ2 windows (clamped into the tile: clamped lanes never store)
template <int IR, int GLOG>
R8B_HD void interp_windows(const FusedParams& p, const TaskGeom<IR, GLOG>& g, const int* __restrict__ s_i, int (&yo)[IQ2])
{
    const int c_cnt = s_i[1], wbase = s_i[3];
#pragma unroll
    for (int q = 0; q < IQ2; q++) {
        int c = g.cb + q * TaskGeom<IR, GLOG>::CL;
        if (c > c_cnt) c = c_cnt;
        int li = c * p.in_step + g.o0 + wbase;
        if (li < 0) li = 0;
        if (li > 2 * FM - p.smaxp) li = 2 * FM - p.smaxp;
        yo[q] = li;
    }
}

// The tap loop: group bank [smaxp][IR] (phase r's filter pre-shifted by its window offset and zero-padded,
// so there are no predicates and one base address), IR x IQ2 accumulators.
template <int IR, bool PADV>
R8B_HD void interp_acc(const double* __restrict__ yb, const double* __restrict__ gb, const int (&yo)[IQ2], int smaxp, int ysh,
                       double (&acc)[IR][IQ2])
{
#pragma unroll
    for (int r = 0; r < IR; r++)
#pragma unroll
        for (int q = 0; q < IQ2; q++) acc[r][q] = 0.0;
#pragma unroll 4
    for (int s = 0; s < smaxp; s++) {
        double yv[IQ2];
#pragma unroll
        for (int q = 0; q < IQ2; q++) yv[q] = PADV ? yb[ylay(yo[q] + s, ysh)] : yb[yo[q] + s];
#pragma unroll
        for (int r = 0; r < IR; r += 2) {
            const double2 b = *reinterpret_cast<const double2*>(gb + s * IR + r);
#pragma unroll
            for (int q = 0; q < IQ2; q++) {
                acc[r][q] = fma(b.x, yv[q], acc[r][q]);
                acc[r + 1][q] = fma(b.y, yv[q], acc[r + 1][q]);
            }
        }
    }
}

// Stores straight from the lane's registers (any IR, ring or linear destination).
template <int IR, int GLOG>
R8B_HD void interp_store_direct(const FusedParams& p, const DstView& dst, int ch, const TaskGeom<IR, GLOG>& g,
                                const int* __restrict__ s_i, double* s_o, const double (&acc)[IR][IQ2])
{
    const int n_j = s_i[0], c_cnt = s_i[1], jshift = s_i[2];
    if (!g.gvalid) return;
#pragma unroll
    for (int q = 0; q < IQ2; q++) {
        const int c = g.cb + q * TaskGeom<IR, GLOG>::CL;
        if (c > c_cnt) continue;
        const int j0 = c * p.out_step + g.r0 + jshift; // relative to the tile's first output
        const bool full = (p.wrap || g.r0 + IR <= p.out_step) && j0 >= 0 && j0 + IR <= n_j;
        if (dst.mask == -1) {
            double* o = s_o + j0;
            if (full && (reinterpret_cast<unsigned long long>(o) & 15) == 0) {
#pragma unroll
                for (int r = 0; r < IR; r += 2) *reinterpret_cast<double2*>(o + r) = make_double2(acc[r][q], acc[r + 1][q]);
            } else {
#pragma unroll
                for (int r = 0; r < IR; r++)
                    if ((p.wrap || g.r0 + r < p.out_step) && j0 + r >= 0 && j0 + r < n_j) o[r] = acc[r][q];
            }
        } else { // ring destination (another stage follows): s_o is the ring slot of the tile's first output
            double* const rb = dst.ptr + (long long) ch * dst.stride;
            const long long i0 = (s_o - rb) + (long long) j0;
#pragma unroll
            for (int r = 0; r < IR; r++)
                if ((p.wrap || g.r0 + r < p.out_step) && j0 + r >= 0 && j0 + r < n_j) rb[(i0 + r) & dst.mask] = acc[r][q];
        }
    }
}

// ---- interpolation on the fp64 tensor path (mma.sync m16n8k16 = SASS DMMA.16x8x16) --------------------------------
// One phase group is a small GEMM: out[c][r] = sum_s Y[c][s] * Bp[s][r], with Y[c][s] = y[c*in_step + o0 + s] a
// strided (Hankel) view of the tile's 2x-rate stream, Bp the group's pre-shifted zero-padded filters [smaxp][8],
// c the stepping cycle, r the phase within the group.  An M tile is 16 stepping cycles; K is taken in chunks of 16 taps
// (m16n8k16), the remainder smaxp % 16 as one m16n8k8 and/or one m16n8k4 product.  Fragments, with g = lane/4,
// t = lane%4: A element a_i = A[g + 8 (i%2)][t + 4 (i/2)]; B element b_i = B[t + 4 i][g]; C element c_i =
// C[g + 8 (i/2)][2t + i%2] -- i.e. a lane ends up with two CONSECUTIVE outputs of each of two stepping cycles and
// four lanes hold one 64-byte output row, so results go straight from the accumulators to global memory with no
// transposition.  Each loaded Y value feeds 8 products, each Bp value 8 mbu, and 2048 multiply-adds issue as one
// instruction.  Every shape accumulates as ONE ascending FMA chain from C over k (tools/mb_dmma_order.cu, bit for bit),
// so a unit's outputs are the plain tap-ascending FMA sums whatever the chunking -- the same as a chain of m8n8k4
// products over 4-tap K-steps, block by block (the CPU emulation computes it that way).  A work unit = one group x mbu
// (2, 4 or 6) blocks of 8 stepping cycles = mbu/2 M tiles.
//
// Which stepping cycle a fragment row stands for is free.  An LDS.64 is served one half-warp at a time, and the
// four rows of a half-warp (4 consecutive doubles each) are conflict-free exactly when their starts are 4 or 12
// doubles apart mod 16.  Windows of cycles kappa apart start kappa*in_step doubles apart, and for every odd in_step
// kappa = 4 gives 4*in_step = 4 or 12 (mod 16): so the rows of a half-warp take cycles 4 apart.  Rows 0..7 and 8..15 of
// an M tile are two "blocks" of 8 rows that interleave to cover 16 consecutive cycles:
//     cycle(block, row) = 16*(block/2) + 4*(row%4) + 2*(block%2) + row/4      (M tile m = blocks 2m, 2m+1)
// (Even in_step: the padded y layout makes the stride odd on average; the same map is used.)
constexpr int MBU_MAX = 6; // blocks per work unit: 2, 4 or 6 (whole M tiles), chosen per call (FusedParams::mbu; fused2_choose_mbu())
R8B_HD int mma_mbu(const FusedParams& p) { return p.mbu >= 2 && p.mbu <= MBU_MAX && (p.mbu & 1) == 0 ? p.mbu : MBU_MAX; }

R8B_HD int mma_cycle(int block, int row) { return 16 * (block >> 1) + 4 * (row & 3) + 2 * (block & 1) + (row >> 2); }

R8B_HD int mma_units(const FusedParams& p, int c_cnt)
{
    const int n_groups = (p.out_step + 7) / 8, n_mb = 2 * (c_cnt / 16 + 1);
    const int mbu = mma_mbu(p);
    return n_groups * ((n_mb + mbu - 1) / mbu);
}

// A work unit's place in the tile: its phase group and which mbu blocks of cycles it covers.  Units are dealt to the
// warps of a half round-robin, so the pair (group, chunk) advances without a division.
struct MmaUnit {
    int g, chunk;
    R8B_HD void set(int unit, int n_groups)
    {
        chunk = unit / n_groups;
        g = unit - chunk * n_groups;
    }
    R8B_HD void advance(int by, int n_groups)
    {
        g += by;
        while (g >= n_groups) {
            g -= n_groups;
            chunk++;
        }
    }
};

// Tile-level values every unit needs (read once per tile from the bookkeeping interp_prepare() left in shared memory)
struct MmaTile {
    int n_j, c_cnt, jshift, wbase;
    long long elem0; // element index of the tile's first output in a typed linear destination
    R8B_HD void load(const int* __restrict__ s_i)
    {
        n_j = s_i[0];
        c_cnt = s_i[1];
        jshift = s_i[2];
        wbase = s_i[3];
        elem0 = (long long) (unsigned int) s_i[4] | ((long long) s_i[5] << 32);
    }
    // from the call's tile table; row = ch * dst.stride
    R8B_HD void load(const TileEntry& e, long long row)
    {
        n_j = e.s[0];
        c_cnt = e.s[1];
        jshift = e.s[2];
        wbase = e.s[3];
        elem0 = row + e.off;
    }
};

// y index (before the padded-layout map) of the lane's A elements of block i (< mbu) of the unit at tap 0: element a_j
// of M tile m (blocks 2m, 2m+1) of the chunk at k0 is at mma_a_index(.., 2m + j%2, ..) + k0 + 4 (j/2)
R8B_HD int mma_a_index(const FusedParams& p, const MmaTile& mt, const MmaUnit& u, int goff, int i, int lane)
{
    int c = mma_cycle(u.chunk * mma_mbu(p) + i, lane >> 2);
    if (c > mt.c_cnt) c = mt.c_cnt;          // rows past the last cycle compute something valid and never store
    int li = c * p.in_step + goff + mt.wbase;
    if (li < 0) li = 0;
    if (li > p.ylen - p.smaxp) li = p.ylen - p.smaxp;
    return li + (lane & 3);
}

// offset of the lane's B element at tap 0 inside the call's bank: b_i = Bp[k0 + lane%4 + 4 i][lane/4] of the chunk at k0
// sits 8 k0 + 32 i further (tensor-path bank layout: within a 4-tap K-step the 32 values sit in fragment order, element
// n*4 + k = Bp[4 ks + k][n])
R8B_HD int mma_b_index(const FusedParams& p, const MmaUnit& u, int lane) { return u.g * p.smaxp * 8 + lane; }

// the lane's two results of block i (< mbu) of the unit: outputs (cycle, phases 2*(lane%4), +1) of the group.
// LIN: the destination is known to be linear fp64 (dst.fmt == FMT_F64, dst.mask == -1), so only that branch is compiled.
template <bool LIN = false>
R8B_HD void mma_store(const FusedParams& p, const DstView& dst, int ch, const MmaTile& mt, double* s_o, const MmaUnit& u, int i, int lane,
                      double c0, double c1)
{
    const int c = mma_cycle(u.chunk * mma_mbu(p) + i, lane >> 2);
    if (c > mt.c_cnt) return;
    const int rr = p.delta + u.g * 8 + 2 * (lane & 3);
    const int j = c * p.out_step + rr + mt.jshift;
    const bool in0 = (p.wrap || rr < p.out_step) && j >= 0 && j < mt.n_j;
    const bool in1 = (p.wrap || rr + 1 < p.out_step) && j + 1 >= 0 && j + 1 < mt.n_j;
    if (!LIN && dst.fmt != FMT_F64) { // narrow on the way out (linear destinations only): the casts of oneshot<Tin,Tout>()
        if (in0) typed_store(dst.ptr, mt.elem0 + j, dst.fmt, dst.scale, c0, dst.dither, dst.stride, dst.base, dst.dither_ch0);
        if (in1) typed_store(dst.ptr, mt.elem0 + j + 1, dst.fmt, dst.scale, c1, dst.dither, dst.stride, dst.base, dst.dither_ch0);
    } else if (LIN || dst.mask == -1) {
        double* o = s_o + j;
        if (in0 && in1 && (reinterpret_cast<unsigned long long>(o) & 15) == 0) {
            *reinterpret_cast<double2*>(o) = make_double2(c0, c1);
        } else {
            if (in0) o[0] = c0;
            if (in1) o[1] = c1;
        }
    } else { // ring destination (another stage follows): s_o is the ring slot of the tile's first output
        double* const rb = dst.ptr + (long long) ch * dst.stride;
        const long long i0 = (s_o - rb) + (long long) j;
        if (in0) rb[i0 & dst.mask] = c0;
        if (in1) rb[(i0 + 1) & dst.mask] = c1;
    }
}

} // namespace f2

} // namespace r8bgpu

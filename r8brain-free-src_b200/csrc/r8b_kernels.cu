// r8b_kernels.cu -- hand-written sm_90a kernels for the CDSPResampler::process() hot path.
//
// Every kernel processes ALL channels of a batch in one launch (channel = outer grid
// dimension); streams are addressed by absolute sample index (see r8b_plan.h), so a kernel
// is a pure function of (history ring, current input block) -> (output range).
//
//   k_blockconv   CDSPBlockConvolver::process + CDSPRealFFT fwd/inv + multiplyBlocksZP +
//                 mirrorInputSpectrum  (CDSPBlockConvolver.h:252-354,606-629; CDSPRealFFT.h:98-385)
//   k_bcl_gather, k_bcl_conv, k_bcl_scatter
//                 the same for low-pass kernels too long for one CTA's tile (r8b_bclarge.cuh)
//   k_frac<false> CDSPFracInterpolator::convolve0<N>      (CDSPFracInterpolator.h:991-1060)
//   k_frac<true>  CDSPFracInterpolator::convolve2          (CDSPFracInterpolator.h:1069-1179)
//   k_hbup        CDSPHBUpsampler::process / convolveN     (CDSPHBUpsampler.h:674-732, .inc)
//   k_hbdown      CDSPHBDownsampler::process / convolveN   (CDSPHBDownsampler.h:137-239, .inc)
//
// fp64 throughout; no tensor cores (1-D convolution, not a dense contraction).
#include "r8b_kernels.h"

#include <climits>

#include "r8b_bclarge.cuh"
#include "r8b_dsd.cuh"
#include "r8b_fft.cuh"
#include "r8b_fused_common.cuh"
#include "r8b_interp.cuh"
#include "r8b_hbfuse.cuh"

namespace r8bgpu {

__device__ __forceinline__ double src_read(const SrcView& v, int ch, long long n)
{
    if (n >= v.avail) return 0.0;
    if (n >= v.cur_base) return __ldg(v.cur + (long long) ch * v.cur_stride + (n - v.cur_base));
    return __ldg(v.ring + (long long) ch * v.ring_stride + (n & v.ring_mask));
}

// src_read for a caller's block of planar DSD bytes (the half-band decimators' DSD instantiations): the block is decoded
// bit by bit, the history ring is read as it is.
__device__ __forceinline__ double src_read_dsd(const SrcView& v, int ch, long long n)
{
    if (n >= v.avail) return 0.0;
    if (n >= v.cur_base)
        return dsd_load(reinterpret_cast<const unsigned char*>(v.cur) + (long long) ch * v.cur_stride, n - v.cur_base,
                        v.cur_fmt == FMT_DSD_MSB, v.cur_scale);
    return __ldg(v.ring + (long long) ch * v.ring_stride + (n & v.ring_mask));
}

// DSD stream-0 loads of the half-band decimators: the window's (even, odd) sample pairs from a caller's block that holds
// the whole window, split straight into the two arrays.  Pair i is the samples a0 + 2i and a0 + 2i + 1 (absolute index
// a0 = 2 * j0 even); put(i, even, odd) stores them.  At odd block starts the two bits of a pair can sit in two bytes.
template <int NT, typename Put>
__device__ __forceinline__ void dsd_pairs(const SrcView& src, int ch, long long a0, int np, int tid, Put put)
{
    const unsigned char* row = reinterpret_cast<const unsigned char*>(src.cur) + (long long) ch * src.cur_stride;
    const bool msb = src.cur_fmt == FMT_DSD_MSB;
    const long long r0 = a0 - src.cur_base; // block index of pair 0's even sample
    for (int i = tid; i < np; i += NT) {
        const long long r = r0 + 2 * i;
        const unsigned char v = __ldg(row + (r >> 3));
        const unsigned char w = ((r + 1) & 7) ? v : __ldg(row + ((r + 1) >> 3)); // one load unless the pair straddles
        put(i, dsd_value(v, r, msb, src.cur_scale), dsd_value(w, r + 1, msb, src.cur_scale));
    }
}

__device__ __forceinline__ void dst_write(const DstView& v, int ch, long long idx, double x)
{
    v.ptr[(long long) ch * v.stride + ((idx - v.base) & v.mask)] = x;
}

// ------------------------------------------------------------------------------------------
// Overlap-save FIR with built-in xU / :D.
//
// Polyphase view of "zero-stuff by U, filter with h, keep every D-th":
//     y[U*m + r] = sum_j g_r[j] * x[m - j],   g_r[j] = h[U*j + r]
// One CTA transforms TWO consecutive tiles (a,b) of one channel packed as z = x_a + i*x_b with a
// single M-point complex FFT.
//   U == 1: g real  =>  IFFT(Z .* G) = y_a + i*y_b                      (1 inverse for 2 tiles)
//   U == 2: G = FFT(g_0 + i*g_1); X_a = (Z[k] + conj Z[M-k])/2, X_b = (Z[k] - conj Z[M-k])/(2i);
//           IFFT(X_t .* G)[m] = y_t[2m] + i*y_t[2m+1]  -- i.e. the inverse transform's interleaved
//           re/im IS the 2x-rate output stream (this replaces mirrorInputSpectrum + the
//           double-length inverse real FFT of the reference).
// Tile geometry: window of M inputs starting at (first valid m) - lg; outputs are valid for
// local positions [lg, M - lg).
// Per-channel call fields of a ragged launch (RaggedRec); the uniform fields describe the largest channel.
__device__ __forceinline__ void ragged_views(const RaggedRec& r, SrcView& src, DstView& dst)
{
    src.cur_base = r.cur_base;
    src.avail = r.avail;
    dst.base = r.dst_base;
}

template <int M, int UP, int NT, bool RAG>
__global__ void __launch_bounds__(NT) k_blockconv(BlockConvParams p, SrcView src, DstView dst, const RaggedRec* __restrict__ rr)
{
    extern __shared__ double2 smem[];
    constexpr int PL = fft_padded_len(M);
    double2* zbuf = smem;
    double2* wbuf = (UP == 2) ? smem + PL : smem;

    const int tid = threadIdx.x;
    const int n_pairs = (p.n_tiles + 1) >> 1;
    const int ch = blockIdx.x / n_pairs;
    const int pair = blockIdx.x - ch * n_pairs;
    const int ta = 2 * pair;
    if constexpr (RAG) {
        const RaggedRec& r = rr[ch];
        if (ta >= r.n_tiles) return;
        p.m0 = r.m0;
        p.m1 = r.m1;
        p.e0 = r.e0;
        p.e1 = r.e1;
        p.n_tiles = r.n_tiles;
        p.adv = r.adv;
        ragged_views(r, src, dst);
    }
    const bool has_b = (ta + 1) < p.n_tiles;
    const long long ma = p.m0 + (long long) ta * p.adv; // first valid input-rate position of tile a
    const long long mb = ma + p.adv;
    const long long wa = ma - p.lg, wb = mb - p.lg;

    if (p.src_up <= 1) {
        for (int n = tid; n < M; n += NT) {
            const double xa = src_read(src, ch, wa + n);
            const double xb = has_b ? src_read(src, ch, wb + n) : 0.0;
            zbuf[fft_pad(n)] = make_double2(xa, xb);
        }
    } else {
        // Non-power-of-two up-factors (3x): the reference zero-stuffs in the time domain
        // (copyUpsample, CDSPBlockConvolver.h:414-496); same here -- the tile is a window of the
        // zero-stuffed stream, read through a virtual view of the source.
        for (int n = tid; n < M; n += NT) {
            const long long ua = wa + n, ub = wb + n;
            const double xa = (ua >= 0 && ua % p.src_up == 0) ? src_read(src, ch, ua / p.src_up) : 0.0;
            const double xb = (has_b && ub >= 0 && ub % p.src_up == 0) ? src_read(src, ch, ub / p.src_up) : 0.0;
            zbuf[fft_pad(n)] = make_double2(xa, xb);
        }
    }
    __syncthreads();
    fft_forward<M, NT>(zbuf, p.tw, tid);

    const long long t_lo = p.e0 * p.down, t_hi = p.e1 * p.down; // y indices [t_lo, t_hi) are wanted

    if (UP == 1) {
        // Power-of-two decimation, reference-exact: the short inverse FFT of the reference sees the
        // low 1/D of the spectrum (spec[] is zero elsewhere) plus one real "Nyquist" value
        // kb[z]*p[z] - kb[z+1]*p[z+1] = H(fs/2D) * (Re X - Im X) (CDSPBlockConvolver.h:329-342 with the
        // zero-phase kernel layout).  In the full-length inverse sampled at multiples of D that value
        // is a component at bin M/(2D); for the packed pair it is (c_a + i*c_b).
        __shared__ double2 nyq;
        const int kq = M / (2 * (p.trunc > 0 ? p.trunc : 1));
        if (p.trunc > 0 && tid == 0) {
            const double2 z1 = zbuf[fft_pad(slot_of<M>(kq))];
            const double2 z2 = zbuf[fft_pad(slot_of<M>(M - kq))];
            const double2 xa = make_double2(0.5 * (z1.x + z2.x), 0.5 * (z1.y - z2.y));
            const double2 xb = make_double2(0.5 * (z1.y + z2.y), 0.5 * (z2.x - z1.x));
            nyq = make_double2(p.nyq_gain * (xa.x - xa.y), p.nyq_gain * (xb.x - xb.y));
        }
        if (p.trunc > 0) __syncthreads();
        const int sq = slot_of<M>(kq);
        for (int s = tid; s < M; s += NT) {
            const double2 z = zbuf[fft_pad(s)];
            const double2 g = __ldg(&p.spec[s]);
            zbuf[fft_pad(s)] = (p.trunc > 0 && s == sq) ? nyq : cmul<+1>(z, g);
        }
        __syncthreads();
        fft_inverse<M, NT>(zbuf, p.tw, tid);
        const double* yb = reinterpret_cast<const double*>(zbuf);
#pragma unroll 1
        for (int which = 0; which < 2; which++) {
            if (which == 1 && !has_b) break;
            const long long mt = which ? mb : ma;
            long long cnt = p.m1 - mt;
            if (cnt > p.adv) cnt = p.adv;
            for (int i = tid; i < cnt; i += NT) {
                const long long t = mt + i;
                if (t < t_lo || t >= t_hi) continue;
                if (p.down > 1 && (t % p.down) != 0) continue;
                dst_write(dst, ch, t / p.down, yb[2 * fft_pad(p.lg + i) + which]);
            }
        }
    } else {
#pragma unroll 1
        for (int which = 0; which < 2; which++) {
            if (which == 1 && !has_b) break;
            for (int s = tid; s < M; s += NT) {
                const int k = freq_of<M>(s);
                const int s2 = slot_of<M>((M - k) & (M - 1));
                const double2 z1 = zbuf[fft_pad(s)];
                const double2 z2 = zbuf[fft_pad(s2)];
                double2 x;
                if (which == 0) x = make_double2(z1.x + z2.x, z1.y - z2.y);       // z1 + conj z2
                else x = make_double2(z1.y + z2.y, z2.x - z1.x);                  // -i (z1 - conj z2)
                wbuf[fft_pad(s)] = cmul<+1>(x, __ldg(&p.spec[s]));
            }
            __syncthreads();
            fft_inverse<M, NT>(wbuf, p.tw, tid);
            const double* yb = reinterpret_cast<const double*>(wbuf);
            const long long mt = which ? mb : ma;
            long long cnt = p.m1 - mt;
            if (cnt > p.adv) cnt = p.adv;
            for (int i = tid; i < 2 * cnt; i += NT) {
                const int ml = i >> 1, r = i & 1;
                const long long t = 2 * (mt + ml) + r;
                if (t < t_lo || t >= t_hi) continue;
                if (p.down > 1 && (t % p.down) != 0) continue;
                dst_write(dst, ch, t / p.down, yb[2 * fft_pad(p.lg + ml) + r]);
            }
            __syncthreads();
        }
    }
}

int blockconv_smem_bytes(int fft_log2, int up)
{
    const int m = 1 << fft_log2;
    return fft_padded_len(m) * (int) sizeof(double2) * (up == 2 ? 2 : 1);
}

template <int M, int UP>
static void launch_bc_inst(const BlockConvParams& p, const SrcView& src, const DstView& dst, int n_ch,
                           cudaStream_t st, const RaggedRec* rr)
{
    constexpr int NT = 256;
    const int smem = blockconv_smem_bytes(p.fft_log2, UP);
    const int n_pairs = (p.n_tiles + 1) >> 1;
    if (rr != nullptr) {
        ensure_dyn_smem<k_blockconv<M, UP, NT, true>>(smem);
        k_blockconv<M, UP, NT, true><<<(unsigned) (n_pairs * n_ch), NT, smem, st>>>(p, src, dst, rr);
        return;
    }
    ensure_dyn_smem<k_blockconv<M, UP, NT, false>>(smem);
    k_blockconv<M, UP, NT, false><<<(unsigned) (n_pairs * n_ch), NT, smem, st>>>(p, src, dst, nullptr);
}

void launch_blockconv(const BlockConvParams& p, const SrcView& src, const DstView& dst, int n_ch,
                      cudaStream_t st, const RaggedRec* rr)
{
    if (p.n_tiles <= 0 || n_ch <= 0) return;
    if (p.up == 1) {
        switch (p.fft_log2) {
        case 6: launch_bc_inst<64, 1>(p, src, dst, n_ch, st, rr); break;   // short kernels, reference-exact decimation
        case 7: launch_bc_inst<128, 1>(p, src, dst, n_ch, st, rr); break;
        case 8: launch_bc_inst<256, 1>(p, src, dst, n_ch, st, rr); break;
        case 9: launch_bc_inst<512, 1>(p, src, dst, n_ch, st, rr); break;
        case 10: launch_bc_inst<1024, 1>(p, src, dst, n_ch, st, rr); break;
        case 11: launch_bc_inst<2048, 1>(p, src, dst, n_ch, st, rr); break;
        case 13: launch_bc_inst<8192, 1>(p, src, dst, n_ch, st, rr); break; // 1x stages only (one buffer)
        default: launch_bc_inst<4096, 1>(p, src, dst, n_ch, st, rr); break;
        }
    } else {
        switch (p.fft_log2) {
        case 10: launch_bc_inst<1024, 2>(p, src, dst, n_ch, st, rr); break;
        case 11: launch_bc_inst<2048, 2>(p, src, dst, n_ch, st, rr); break;
        default: launch_bc_inst<4096, 2>(p, src, dst, n_ch, st, rr); break;
        }
    }
}

cudaError_t blockconv_configure() { return cudaSuccess; }

// ------------------------------------------------------------------------------------------
// Large-tile overlap-save (M = 16384 .. 65536): three launches through an HBM scratch buffer, per-thread steps in
// r8b_bclarge.cuh.  Grid of the gather / scatter kernels: (channel, pair) units x 4096 / ITEM_NT CTAs; consecutive
// threads take consecutive n1, so every load and store of a warp is one contiguous run.
template <int R0>
__global__ void __launch_bounds__(bcl::ITEM_NT) k_bcl_gather(const __grid_constant__ BcLargeParams p, const __grid_constant__ SrcView src)
{
    constexpr int CPU = bcl::SUB / bcl::ITEM_NT; // CTAs per unit
    const int unit = blockIdx.x / CPU;
    const int n1 = (blockIdx.x - unit * CPU) * bcl::ITEM_NT + threadIdx.x;
    const bcl::Pair t = bcl::pair_of(p.bc, unit);
    bcl::gather_item<R0>(p, src, t, n1, p.scratch + (long long) unit * R0 * bcl::SUB);
}

template <int R0>
__global__ void __launch_bounds__(bcl::ITEM_NT) k_bcl_scatter(const __grid_constant__ BcLargeParams p, const __grid_constant__ DstView dst)
{
    constexpr int CPU = bcl::SUB / bcl::ITEM_NT;
    const int unit = blockIdx.x / CPU;
    const int n1 = (blockIdx.x - unit * CPU) * bcl::ITEM_NT + threadIdx.x;
    const bcl::Pair t = bcl::pair_of(p.bc, unit);
    bcl::scatter_item<R0>(p, dst, t, n1, p.scratch + (long long) unit * R0 * bcl::SUB);
}

// Ragged forms: unit = channel * (largest channel's pairs) + pair; a unit past its channel's pairs exits at once (the
// conv kernel transforms its scratch block anyway: nothing reads it).
__device__ __forceinline__ bool bcl_ragged_unit(const BcLargeParams& p, const RaggedRec* __restrict__ rr, int unit,
                                                BcLargeParams& q, bcl::Pair& t, int& ch)
{
    const int np = bcl::n_pairs(p.bc);
    ch = unit / np;
    const int pr = unit - ch * np;
    const RaggedRec& r = rr[ch];
    if (2 * pr >= r.n_tiles) return false;
    q = p;
    q.bc.m0 = r.m0;
    q.bc.m1 = r.m1;
    q.bc.e0 = r.e0;
    q.bc.e1 = r.e1;
    q.bc.n_tiles = r.n_tiles;
    q.bc.adv = r.adv;
    t = bcl::pair_of(q.bc, pr);
    t.ch = ch;
    return true;
}

template <int R0>
__global__ void __launch_bounds__(bcl::ITEM_NT) k_bcl_gather_ragged(const __grid_constant__ BcLargeParams p,
                                                                    const __grid_constant__ SrcView src,
                                                                    const RaggedRec* __restrict__ rr)
{
    constexpr int CPU = bcl::SUB / bcl::ITEM_NT;
    const int unit = blockIdx.x / CPU;
    const int n1 = (blockIdx.x - unit * CPU) * bcl::ITEM_NT + threadIdx.x;
    BcLargeParams q;
    bcl::Pair t;
    int ch;
    if (!bcl_ragged_unit(p, rr, unit, q, t, ch)) return;
    SrcView s = src;
    DstView unused{};
    ragged_views(rr[ch], s, unused);
    bcl::gather_item<R0>(q, s, t, n1, p.scratch + (long long) unit * R0 * bcl::SUB);
}

template <int R0>
__global__ void __launch_bounds__(bcl::ITEM_NT) k_bcl_scatter_ragged(const __grid_constant__ BcLargeParams p,
                                                                     const __grid_constant__ DstView dst,
                                                                     const RaggedRec* __restrict__ rr)
{
    constexpr int CPU = bcl::SUB / bcl::ITEM_NT;
    const int unit = blockIdx.x / CPU;
    const int n1 = (blockIdx.x - unit * CPU) * bcl::ITEM_NT + threadIdx.x;
    BcLargeParams q;
    bcl::Pair t;
    int ch;
    if (!bcl_ragged_unit(p, rr, unit, q, t, ch)) return;
    DstView d = dst;
    SrcView unused{};
    ragged_views(rr[ch], unused, d);
    bcl::scatter_item<R0>(q, d, t, n1, p.scratch + (long long) unit * R0 * bcl::SUB);
}

// one CTA per (unit, sub-block r): 4096-point forward transform, filter, inverse, in shared memory
template <int NT>
__global__ void __launch_bounds__(NT) k_bcl_conv(const __grid_constant__ BcLargeParams p)
{
    extern __shared__ double2 smem[];
    __shared__ double2 nyq;
    const int tid = threadIdx.x;
    const int r0 = 1 << (p.bc.fft_log2 - 12);
    const int r = blockIdx.x & (r0 - 1);
    double2* __restrict__ blk = p.scratch + (long long) blockIdx.x * bcl::SUB; // unit * M + r * 4096
    for (int n = tid; n < bcl::SUB; n += NT) smem[fft_pad(n)] = blk[n];
    __syncthreads();
    fft_forward<bcl::SUB, NT>(smem, p.bc.tw, tid);
    const bool nyq_here = p.bc.trunc > 0 && r == 0;
    if (nyq_here) {
        if (tid == 0) nyq = bcl::conv_nyquist(p, smem);
        __syncthreads();
    }
    for (int s = tid; s < bcl::SUB; s += NT) bcl::conv_mul_item(p, smem, r, s, nyq_here, nyq);
    __syncthreads();
    fft_inverse<bcl::SUB, NT>(smem, p.bc.tw, tid);
    for (int n = tid; n < bcl::SUB; n += NT) blk[n] = smem[fft_pad(n)];
}

template <int R0>
static void launch_bcl_group(const BcLargeParams& p, const SrcView& src, const DstView& dst, int nch, cudaStream_t st,
                             const RaggedRec* rr)
{
    constexpr int NT = 256;
    constexpr int smem = bcl::SUB_PL * (int) sizeof(double2);
    ensure_dyn_smem<k_bcl_conv<NT>>(smem);
    const unsigned units = (unsigned) (bcl::n_pairs(p.bc) * nch);
    if (rr != nullptr) {
        k_bcl_gather_ragged<R0><<<units * (bcl::SUB / bcl::ITEM_NT), bcl::ITEM_NT, 0, st>>>(p, src, rr);
        k_bcl_conv<NT><<<units * R0, NT, smem, st>>>(p);
        k_bcl_scatter_ragged<R0><<<units * (bcl::SUB / bcl::ITEM_NT), bcl::ITEM_NT, 0, st>>>(p, dst, rr);
        return;
    }
    k_bcl_gather<R0><<<units * (bcl::SUB / bcl::ITEM_NT), bcl::ITEM_NT, 0, st>>>(p, src);
    k_bcl_conv<NT><<<units * R0, NT, smem, st>>>(p);
    k_bcl_scatter<R0><<<units * (bcl::SUB / bcl::ITEM_NT), bcl::ITEM_NT, 0, st>>>(p, dst);
}

int launch_blockconv_large(const BcLargeParams& p, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st,
                           const RaggedRec* rr)
{
    if (p.bc.n_tiles <= 0 || n_ch <= 0) return 0;
    int launches = 0;
    for (int c0 = 0; c0 < n_ch; c0 += p.group_ch) {
        const int nch = n_ch - c0 < p.group_ch ? n_ch - c0 : p.group_ch;
        SrcView s = src;
        s.ring += (long long) c0 * s.ring_stride;
        if (s.cur != nullptr) s.cur += (long long) c0 * s.cur_stride;
        DstView d = dst;
        d.ptr += (long long) c0 * d.stride;
        const RaggedRec* r = rr != nullptr ? rr + c0 : nullptr;
        switch (p.bc.fft_log2) {
        case 14: launch_bcl_group<4>(p, s, d, nch, st, r); break;
        case 15: launch_bcl_group<8>(p, s, d, nch, st, r); break;
        default: launch_bcl_group<16>(p, s, d, nch, st, r); break;
        }
        launches += 3;
    }
    return launches;
}

// ------------------------------------------------------------------------------------------
// Fractional-delay interpolation.  One block = `tile` consecutive outputs of one channel; the input
// window they touch is staged once in shared memory (positions are non-decreasing in the output
// index, so the window is [pos(first) - fll, pos(last) - fll + flen)).
//
// Whole-number stepping: output j sits at input position j*InStep/OutStep; the fractional part selects
// one of OutStep precomputed filters.
// Non-whole stepping: bank of `fracs` filters, each tap a quadratic in the residual fraction.  The
// timing arithmetic reproduces the reference's IEEE expression order exactly
// ((InCounter + InPosShift) * ssr) / dsr -- explicit _rn intrinsics forbid FMA contraction.
template <bool POLY>
__device__ __forceinline__ void frac_position(const FracParams& p, long long k, long long& ip, int& phase,
                                              double& fpos)
{
    if (!POLY) {
        const long long pos = (p.e0 + k) * p.in_step;
        ip = pos / p.out_step;
        phase = (int) (pos - ip * p.out_step);
        fpos = 0.0;
        return;
    }
    phase = 0;
    ip = p.p0;
    fpos = p.fpos0;
    if (p.pos_dp != nullptr) { // R8B_FASTTIMING: host-walked sequence
        ip = p.p0 + __ldg(p.pos_dp + k);
        fpos = __ldg(p.pos_fpos + k);
    } else if (k > 0) {
        const int ic = p.in_counter0 + (int) k;
        const double np = __ddiv_rn(__dmul_rn(__dadd_rn((double) ic, p.in_pos_shift), p.ssr), p.dsr);
        const int ni = __double2int_rz(np);
        ip = p.p0 + (ni - p.in_pos_int0);
        fpos = __dsub_rn(np, (double) ni);
    }
}

template <bool POLY, bool RAG>
__global__ void __launch_bounds__(256) k_frac(FracParams p, SrcView src, DstView dst, int tile, int cap,
                                              const RaggedRec* __restrict__ rr)
{
    extern __shared__ double s_x[];
    const int ch = blockIdx.y, tid = threadIdx.x;
    const long long k0 = (long long) blockIdx.x * tile;
    if constexpr (RAG) {
        const RaggedRec& r = rr[ch];
        if (k0 >= r.e1 - r.e0) return;
        p.e0 = r.e0;
        p.e1 = r.e1;
        p.in_counter0 = r.in_counter0;
        p.in_pos_int0 = r.in_pos_int0;
        p.in_pos_shift = r.in_pos_shift;
        p.fpos0 = r.fpos0;
        p.p0 = r.p0;
        if constexpr (POLY) { // the host's doubles, as they are: the position expression stays bit-exact
            p.ssr = r.ssr;
            p.dsr = r.dsr;
        }
        ragged_views(r, src, dst);
    }
    const int cnt = (int) min((long long) tile, p.e1 - p.e0 - k0);
    long long ip_lo, ip_hi;
    int ph;
    double fp;
    frac_position<POLY>(p, k0, ip_lo, ph, fp);
    frac_position<POLY>(p, k0 + cnt - 1, ip_hi, ph, fp);
    const int len = (int) (ip_hi - ip_lo) + p.flen;
    if (len > cap) __trap(); // host sizing bug; never silently wrong
    const long long base = ip_lo - p.fll;
    for (int i = tid; i < len; i += 256) s_x[i] = src_read(src, ch, base + i);
    __syncthreads();
    for (int kk = tid; kk < cnt; kk += 256) {
        long long ip;
        frac_position<POLY>(p, k0 + kk, ip, ph, fp);
        const double* __restrict__ xs = s_x + (int) (ip - ip_lo);
        double acc = 0.0;
        if (!POLY) {
            const double* __restrict__ b = p.bank + (long long) ph * p.flen;
            for (int i = 0; i < p.flen; i++) acc = fma(__ldg(b + i), xs[i], acc);
        } else {
            double x = __dmul_rn(fp, (double) p.fracs);
            const int fti = __double2int_rz(x);
            x = __dsub_rn(x, (double) fti);
            const double x2 = __dmul_rn(x, x);
            acc = poly_row_dot<false>(p.bank + (long long) fti * p.flen * 3, p.flen, x, x2, [=](int i) { return xs[i]; });
        }
        dst_write(dst, ch, p.e0 + k0 + kk, acc);
    }
}

template <bool POLY>
static void launch_frac(const FracParams& p, int tile, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st,
                        const RaggedRec* rr)
{
    const long long n = p.e1 - p.e0;
    if (n <= 0 || n_ch <= 0) return;
    dim3 grid((unsigned) ((n + tile - 1) / tile), (unsigned) n_ch);
    if (rr != nullptr) k_frac<POLY, true><<<grid, 256, FRAC_CAP * sizeof(double), st>>>(p, src, dst, tile, FRAC_CAP, rr);
    else k_frac<POLY, false><<<grid, 256, FRAC_CAP * sizeof(double), st>>>(p, src, dst, tile, FRAC_CAP, nullptr);
}

void launch_frac_whole(const FracParams& p, int tile, const SrcView& src, const DstView& dst, int n_ch,
                       cudaStream_t st, const RaggedRec* rr)
{
    launch_frac<false>(p, tile, src, dst, n_ch, st, rr);
}

void launch_frac_poly(const FracParams& p, int tile, const SrcView& src, const DstView& dst, int n_ch,
                      cudaStream_t st, const RaggedRec* rr)
{
    launch_frac<true>(p, tile, src, dst, n_ch, st, rr);
}

// ------------------------------------------------------------------------------------------
// Half-band 2x upsampler: even outputs copy the input, odd outputs are the symmetric FIR.
template <bool RAG>
__global__ void __launch_bounds__(256) k_hbup(HbParams p, SrcView src, DstView dst, const RaggedRec* __restrict__ rr)
{
    const int ch = blockIdx.y;
    if constexpr (RAG) {
        const RaggedRec& r = rr[ch];
        p.e0 = r.e0;
        p.e1 = r.e1;
        ragged_views(r, src, dst);
    }
    const long long n = (p.e0 >> 1) + (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (2 * n >= p.e1) return;
    const double c = src_read(src, ch, n);
    double acc = p.taps[0] * (src_read(src, ch, n + 1) + c);
    for (int k = 1; k < p.ntaps; k++)
        acc = fma(p.taps[k], src_read(src, ch, n + 1 + k) + src_read(src, ch, n - k), acc);
    dst_write(dst, ch, 2 * n, c);
    dst_write(dst, ch, 2 * n + 1, acc);
}

void launch_hbup(const HbParams& p, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st, const RaggedRec* rr)
{
    const long long n = (p.e1 - p.e0) / 2;
    if (n <= 0 || n_ch <= 0) return;
    dim3 grid((unsigned) ((n + 255) / 256), (unsigned) n_ch);
    if (rr != nullptr) k_hbup<true><<<grid, 256, 0, st>>>(p, src, dst, rr);
    else k_hbup<false><<<grid, 256, 0, st>>>(p, src, dst, nullptr);
}

// Half-band 2x decimator (gain 2, compensated by the following low-pass's gain).
// One block = HBD_TILE outputs of one channel; its input window is staged once in shared memory,
// split into the even (centre) and odd (tapped) samples so that consecutive lanes read consecutive
// words.  Summation order per output: centre, then taps k = 0..T-1 on (x[c+1+2k] + x[c-1-2k]).
// DSD: the caller's block is planar DSD bytes (SrcView::cur_fmt), decoded in the loads.
constexpr int HBD_TILE = 1024;
template <bool RAG, bool DSD>
__global__ void __launch_bounds__(256) k_hbdown(HbParams p, SrcView src, DstView dst, const RaggedRec* __restrict__ rr)
{
    __shared__ double s_even[HBD_TILE];
    __shared__ double s_odd[HBD_TILE + 2 * 14];
    const int ch = blockIdx.y, tid = threadIdx.x, T = p.ntaps;
    if constexpr (RAG) {
        const RaggedRec& r = rr[ch];
        if ((long long) blockIdx.x * HBD_TILE >= r.e1 - r.e0) return;
        p.e0 = r.e0;
        p.e1 = r.e1;
        ragged_views(r, src, dst);
    }
    const long long m0 = p.e0 + (long long) blockIdx.x * HBD_TILE;
    const int cnt = (int) min((long long) HBD_TILE, p.e1 - m0);
    // s_odd[i] = x[2*(m0 - T + i) + 1], i < cnt + 2T - 1 ; s_even[i] = x[2*(m0 + i)], i < cnt
    const long long n0 = 2 * (m0 - T) + 1;
    const int n_in = 2 * (cnt + 2 * T - 1) - 1;
    // Fast path: the whole window lies in one contiguous, 16-byte aligned run (the caller's block, or the ring without a
    // wrap): sample pairs (x[2j], x[2j+1]) arrive as one 128-bit load and split straight into the two arrays.
    const long long j0 = m0 - T, j1 = m0 + cnt + T - 1; // pairs j0 .. j1-1
    if constexpr (DSD) {
        if (2 * j0 >= src.cur_base && 2 * j1 <= src.avail) {
            dsd_pairs<256>(src, ch, 2 * j0, (int) (j1 - j0), tid, [&](int i, double ev, double od) {
                s_odd[i] = od;
                const int e = i - T;
                if (e >= 0 && e < cnt) s_even[e] = ev;
            });
        } else {
            for (int i = tid; i < n_in; i += 256) {
                const double x = src_read_dsd(src, ch, n0 + i);
                if (i & 1) {
                    const int e = (i + 1) / 2 - T;
                    if (e >= 0 && e < cnt) s_even[e] = x;
                } else {
                    s_odd[i >> 1] = x;
                }
            }
        }
    } else {
        const double* run = nullptr;
        if (2 * j0 >= src.cur_base && 2 * j1 <= src.avail) {
            run = src.cur + (long long) ch * src.cur_stride + (2 * j0 - src.cur_base);
        } else if (j0 >= 0 && 2 * j1 <= src.avail && 2 * j1 <= src.cur_base) {
            const long long i0 = (2 * j0) & src.ring_mask;
            if (i0 + 2 * (j1 - j0) <= src.ring_mask + 1) run = src.ring + (long long) ch * src.ring_stride + i0;
        }
        if (run != nullptr && (reinterpret_cast<unsigned long long>(run) & 15) == 0) {
            const double2* __restrict__ r2 = reinterpret_cast<const double2*>(run);
            const int np = (int) (j1 - j0);
            for (int i = tid; i < np; i += 256) {
                const double2 v = __ldg(r2 + i);
                s_odd[i] = v.y;
                const int e = i - T;
                if (e >= 0 && e < cnt) s_even[e] = v.x;
            }
        } else {
            for (int i = tid; i < n_in; i += 256) {
                const double x = src_read(src, ch, n0 + i);
                if (i & 1) {
                    const int e = (i + 1) / 2 - T; // n0+i = 2*(m0-T) + i+1
                    if (e >= 0 && e < cnt) s_even[e] = x;
                } else {
                    s_odd[i >> 1] = x;
                }
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < cnt; i += 256) {
        double acc = s_even[i];
        for (int k = 0; k < T; k++) acc = fma(p.taps[k], s_odd[i + T + k] + s_odd[i + T - 1 - k], acc);
        dst_write(dst, ch, m0 + i, acc);
    }
}

void launch_hbdown(const HbParams& p, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st, const RaggedRec* rr)
{
    const long long n = p.e1 - p.e0;
    if (n <= 0 || n_ch <= 0) return;
    dim3 grid((unsigned) ((n + HBD_TILE - 1) / HBD_TILE), (unsigned) n_ch);
    if (rr != nullptr) k_hbdown<true, false><<<grid, 256, 0, st>>>(p, src, dst, rr);
    else if (is_dsd_format(src.cur_fmt)) k_hbdown<false, true><<<grid, 256, 0, st>>>(p, src, dst, nullptr);
    else k_hbdown<false, false><<<grid, 256, 0, st>>>(p, src, dst, nullptr);
}

// ------------------------------------------------------------------------------------------
// k_hbdown_cascade -- a run of half-band decimators (CDSPHBDownsampler.h:137-239, chained by CDSPResampler.h:337-346,
// 372-391) in ONE launch.  A CTA owns `w` consecutive outputs of the LAST stage of one channel; the source samples they
// depend on (w * 2^n plus the halo the taps reach through all stages) are read once, every intermediate rate is computed
// into shared memory, only the last stage's outputs leave.  Each stream is kept as two arrays, samples of even and of odd
// absolute index: stage arithmetic  out[m] = x[2m] + sum_k f[k] (x[2m+1+2k] + x[2m-1-2k])  then reads consecutive words
// for consecutive m (E[m] and O[m+k], O[m-1-k]), the layout k_hbdown uses for one stage.  Stream s covers absolute
// indices [lo_s, hi_s):  lo_s = 2 lo_{s+1} - (2 T_s - 1),  hi_s = 2 hi_{s+1} + 2 T_s - 2.  Outputs a stage has not yet
// "emitted" are never needed: an output is emitted exactly when its whole upward reach has arrived (r8b_plan.h), so
// every halo read lies below the source's `avail`; indices below zero read the zero history.  Same summation order per
// output as k_hbdown: centre sample, then taps k = 0..T-1.
// DSD: the caller's block is planar DSD bytes (SrcView::cur_fmt); stream 0 decodes them in its loads.
constexpr int HBDC_NT = 256;
template <bool DSD>
__global__ void __launch_bounds__(HBDC_NT) k_hbdown_cascade(const __grid_constant__ HbDownCascParams p, const __grid_constant__ SrcView src,
                                                            const __grid_constant__ DstView dst)
{
    extern __shared__ double hsm[];
    const int n = p.n_stages, tid = threadIdx.x;
    const int ch = blockIdx.x / p.n_tiles, ti = blockIdx.x - ch * p.n_tiles;
    const long long m0 = p.e0 + (long long) ti * p.w;
    long long m1 = m0 + p.w;
    if (m1 > p.e1) m1 = p.e1;
    if (m1 <= m0) return;
    // stream 0: [lo, hi) = [2^n m0 - back[0], 2^n (m1 - 1) + back[0] + 1)
    {
        const long long lo = (m0 << n) - p.back[0], hi = ((m1 - 1) << n) + p.back[0] + 1;
        double* E = hsm + p.boff[0];
        double* O = E + p.cap[0];
        // element with absolute index a lives at E[(a - lo_e) / 2] (a even) or O[(a - lo_o) / 2] (a odd), lo_e / lo_o the
        // first even / odd index >= lo
        const long long lo_e = lo + (lo & 1), lo_o = lo + 1 - (lo & 1);
        const int cnt = (int) (hi - lo);
        if constexpr (DSD) {
            if (lo >= src.cur_base && hi <= src.avail) { // the caller's block holds the window
                const int lead = (int) (lo_e - lo); // 0 or 1: the odd sample in front of the first pair
                if (lead && tid == 0) O[0] = src_read_dsd(src, ch, lo);
                const int np = (cnt - lead) >> 1;
                const int oo = (int) ((lo_e + 1 - lo_o) >> 1);
                dsd_pairs<HBDC_NT>(src, ch, lo_e, np, tid, [&](int i, double ev, double od) {
                    E[i] = ev;
                    O[oo + i] = od;
                });
                if (((cnt - lead) & 1) && tid == 0) E[np] = src_read_dsd(src, ch, lo_e + 2 * np);
            } else {
                for (int i = tid; i < cnt; i += HBDC_NT) {
                    const long long idx = lo + i;
                    const double x = src_read_dsd(src, ch, idx);
                    if (idx & 1) O[(idx - lo_o) >> 1] = x;
                    else E[(idx - lo_e) >> 1] = x;
                }
            }
        } else {
            // contiguous run holding [lo, hi): the caller's block, or the ring without a wrap
            const double* run = nullptr;
            if (lo >= src.cur_base && hi <= src.avail) {
                run = src.cur + (long long) ch * src.cur_stride + (lo - src.cur_base);
            } else if (lo >= 0 && hi <= src.avail && hi <= src.cur_base) {
                const long long i0 = lo & src.ring_mask;
                if (i0 + cnt <= src.ring_mask + 1) run = src.ring + (long long) ch * src.ring_stride + i0;
            }
            if (run != nullptr) {
                // 128-bit loads of (even, odd) pairs from the first even index on; the odd sample in front of it, if any, alone
                const int lead = (int) (lo_e - lo); // 0 or 1
                if (lead && tid == 0) O[0] = __ldg(run);
                const double* a = run + lead;
                const int np = (cnt - lead) >> 1;
                const int oo = (int) ((lo_e + 1 - lo_o) >> 1); // O index of the odd sample of pair 0
                if ((reinterpret_cast<unsigned long long>(a) & 15) == 0) {
                    const double2* __restrict__ a2 = reinterpret_cast<const double2*>(a);
    #pragma unroll 4
                    for (int i = tid; i < np; i += HBDC_NT) {
                        const double2 v = __ldg(a2 + i);
                        E[i] = v.x;
                        O[oo + i] = v.y;
                    }
                } else {
    #pragma unroll 4
                    for (int i = tid; i < np; i += HBDC_NT) {
                        E[i] = __ldg(a + 2 * i);
                        O[oo + i] = __ldg(a + 2 * i + 1);
                    }
                }
                if (((cnt - lead) & 1) && tid == 0) E[np] = __ldg(a + 2 * np); // a trailing even sample
            } else {
                for (int i = tid; i < cnt; i += HBDC_NT) {
                    const long long idx = lo + i;
                    const double x = src_read(src, ch, idx);
                    if (idx & 1) O[(idx - lo_o) >> 1] = x;
                    else E[(idx - lo_e) >> 1] = x;
                }
            }
        }
    }
    __syncthreads();
    for (int s = 0; s < n; s++) {
        const int T = p.ntaps[s], sh = n - s;
        // input stream s and output stream s + 1 ranges
        const long long ilo = (m0 << sh) - p.back[s];
        const long long olo = (m0 << (sh - 1)) - p.back[s + 1], ohi = ((m1 - 1) << (sh - 1)) + p.back[s + 1] + 1;
        const double* __restrict__ Ei = hsm + p.boff[s];
        const double* __restrict__ Oi = Ei + p.cap[s];
        const long long ilo_e = ilo + (ilo & 1), ilo_o = ilo + 1 - (ilo & 1);
        const bool last = (s + 1 == n);
        double* Eo = last ? nullptr : hsm + p.boff[s + 1];
        double* Oo = last ? nullptr : Eo + p.cap[s + 1];
        const long long olo_e = olo + (olo & 1), olo_o = olo + 1 - (olo & 1);
        const int cnt = (int) (ohi - olo);
        const double* __restrict__ f = p.taps[s];
        for (int i = tid; i < cnt; i += HBDC_NT) {
            const long long m = olo + i;
            // x[2m] = E[(2m - ilo_e)/2]; x[2m+1+2k] = O[(2m + 1 + 2k - ilo_o)/2]; x[2m-1-2k] = O[(2m - 1 - 2k - ilo_o)/2]
            const int ie = (int) ((2 * m - ilo_e) >> 1), io = (int) ((2 * m + 1 - ilo_o) >> 1);
            double acc = Ei[ie];
            for (int k = 0; k < T; k++) acc = fma(f[k], Oi[io + k] + Oi[io - 1 - k], acc);
            if (m < 0) acc = 0.0; // a stage's stream starts at index 0: the next stage sees silence before it
            if (last) dst_write(dst, ch, m, acc);
            else if (m & 1) Oo[(m - olo_o) >> 1] = acc;
            else Eo[(m - olo_e) >> 1] = acc;
        }
        __syncthreads();
    }
}

int hbdown_cascade_plan(HbDownCascParams& p, int smem_budget_doubles)
{
    const int n = p.n_stages;
    p.back[n] = 0;
    for (int s = n - 1; s >= 0; s--) p.back[s] = 2 * p.back[s + 1] + 2 * p.ntaps[s] - 1;
    // widest tile whose buffers fit: stream s holds (w - 1) * 2^(n-s) + 2 back[s] + 1 samples, split in two halves
    int best = 0;
    for (int w = 8; w <= 1024; w *= 2) {
        long long tot = 0;
        for (int s = 0; s < n; s++) tot += 2 * ((((long long) (w - 1) << (n - s)) + 2 * p.back[s] + 1) / 2 + 2);
        if (tot <= smem_budget_doubles) best = w;
    }
    if (best == 0) return 0;
    p.w = best;
    int off = 0;
    for (int s = 0; s < n; s++) {
        p.cap[s] = (int) ((((long long) (best - 1) << (n - s)) + 2 * p.back[s] + 1) / 2 + 2);
        p.boff[s] = off;
        off += 2 * p.cap[s];
    }
    p.boff[n] = off;
    p.cap[n] = 0;
    return off * (int) sizeof(double);
}

void launch_hbdown_cascade(const HbDownCascParams& p, int smem_bytes, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st)
{
    if (p.e1 <= p.e0 || n_ch <= 0 || p.n_tiles <= 0) return;
    const unsigned grid = (unsigned) ((long long) p.n_tiles * n_ch);
    if (is_dsd_format(src.cur_fmt)) {
        ensure_dyn_smem<k_hbdown_cascade<true>>(227 * 1024);
        k_hbdown_cascade<true><<<grid, HBDC_NT, smem_bytes, st>>>(p, src, dst);
        return;
    }
    ensure_dyn_smem<k_hbdown_cascade<false>>(227 * 1024); // opt-in once per device, to the limit: later plans may need more than the first
    k_hbdown_cascade<false><<<grid, HBDC_NT, smem_bytes, st>>>(p, src, dst);
}

// ------------------------------------------------------------------------------------------
// DSD: cur is a planar DSD block that the first kernel decoded in its loads, rows of cur_stride bytes (r8b_dsd.cuh).
template <bool DSD>
__global__ void __launch_bounds__(256) k_save_tail(const double* __restrict__ cur, long long cur_stride,
                                                   long long cur_base, long long n0, long long n1,
                                                   double* __restrict__ ring, long long ring_stride,
                                                   long long ring_mask, int fmt, double scale)
{
    const long long n = n0 + (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n1) return;
    const int ch = blockIdx.y;
    if constexpr (DSD) {
        ring[(long long) ch * ring_stride + (n & ring_mask)] =
            dsd_load(reinterpret_cast<const unsigned char*>(cur) + (long long) ch * cur_stride, n - cur_base, fmt == FMT_DSD_MSB, scale);
        return;
    }
    const long long i = (long long) ch * cur_stride + (n - cur_base);
    ring[(long long) ch * ring_stride + (n & ring_mask)] = fmt == FMT_F64 ? cur[i] : typed_load(cur, i, fmt, scale);
}

void launch_save_tail(const double* cur, long long cur_stride, long long cur_base, long long n0,
                      long long n1, double* ring, long long ring_stride, long long ring_mask, int n_ch,
                      cudaStream_t st, int fmt, double scale)
{
    const long long n = n1 - n0;
    if (n <= 0 || n_ch <= 0) return;
    dim3 grid((unsigned) ((n + 255) / 256), (unsigned) n_ch);
    if (is_dsd_format(fmt)) k_save_tail<true><<<grid, 256, 0, st>>>(cur, cur_stride, cur_base, n0, n1, ring, ring_stride, ring_mask, fmt, scale);
    else k_save_tail<false><<<grid, 256, 0, st>>>(cur, cur_stride, cur_base, n0, n1, ring, ring_stride, ring_mask, fmt, scale);
}

__global__ void __launch_bounds__(256) k_save_tail_ragged(const double* __restrict__ cur, long long cur_stride,
                                                          double* __restrict__ ring, long long ring_stride,
                                                          long long ring_mask, const RaggedRec* __restrict__ rr)
{
    const int ch = blockIdx.y;
    const RaggedRec& r = rr[ch];
    const long long n = r.m0 + (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= r.m1) return;
    ring[(long long) ch * ring_stride + (n & ring_mask)] = cur[(long long) ch * cur_stride + (n - r.cur_base)];
}

void launch_save_tail_ragged(const double* cur, long long cur_stride, long long n, double* ring, long long ring_stride,
                             long long ring_mask, int n_ch, cudaStream_t st, const RaggedRec* rr)
{
    if (n <= 0 || n_ch <= 0) return;
    dim3 grid((unsigned) ((n + 255) / 256), (unsigned) n_ch);
    k_save_tail_ragged<<<grid, 256, 0, st>>>(cur, cur_stride, ring, ring_stride, ring_mask, rr);
}

// ------------------------------------------------------------------------------------------
// Fused cascade of half-band 2x upsamplers (CDSPHBUpsampler chain of e.g. 44100 -> 2822400,
// CDSPResampler.h:207-211): one read of the first stream, one write of the last; every
// intermediate rate lives only in shared memory.  A CTA owns `w` samples of the cascade's input
// stream s0 (plus the halo the taps reach back/forward through all stages) and produces the
// corresponding w * 2^c samples of s_c.
//   s_{k+1}[2n] = s_k[n];  s_{k+1}[2n+1] = sum_j f_k[j] * (s_k[n-j] + s_k[n+1+j]);  s_k[<0] = 0.
#ifndef R8BGPU_HB_NT
#define R8BGPU_HB_NT 128 // CTA shape: see the note at k_hbup_cascade
#endif
constexpr int HB_NT = R8BGPU_HB_NT;
__device__ __forceinline__ int hb_pad(int i) { return i + (i >> 2); }
// Layout of one shared-memory stream buffer: element i at i + (i >> sh).  sh = 2 (hb_pad) suits hb_stage, whose lanes read
// 4 samples apart; the buffer the fused last-two-stages pass reads -- lanes 2 samples apart -- uses sh = 4: with hb_pad its
// loads and the producing stage's stores were both 2-way bank-conflicted (ncu: 4.05 wavefronts per LDS.64 instead of 2).
__device__ __forceinline__ int hb_lay(int i, int sh) { return i + (i >> sh); }

// Final-stream stores of the half-band cascade: a thread owns 8 consecutive outputs (64 B) and writes them as four
// 128-bit stores, Hopper's widest, so one warp store instruction covers half of each of 32 sectors.  Making every
// instruction write whole sectors (the lanes of a pair trading halves by shuffle) was measured slower on H100: cfg 4's
// cascade 3.22 ms against 3.02 ms per step, bit-identical output -- the exchange costs more than the sectors save.

// One cascade stage for a CTA: every thread produces 4 consecutive input positions (8 outputs) from a
// register window of 2T+3 samples -- 2T+3 shared-memory loads instead of 4*2T.  All indices are 32-bit
// tile-local; buffers use the skewed layout i -> i + (i >> 2) so that threads 4 samples apart hit
// different banks (lane stride 5 doubles).  Because (4q + o) >> 2 == q + (o >> 2), every address is
// 5q (loads) / 10q (stores) plus a warp-uniform term.
template <int T>
__device__ __forceinline__ void hb_stage(const double* __restrict__ in, long long in_lo, const double* __restrict__ f,
                                         long long L, long long H, double* __restrict__ out, bool last, int osh,
                                         const HbCascadeParams& p, const DstView& dst, int ch, int tid)
{
    const long long n_lo = (L >= 0) ? L / 2 : -((-L + 1) / 2);               // floor(L/2)
    const long long n_hi = (H - 1 >= 0) ? (H - 1) / 2 : -((-(H - 1) + 1) / 2); // floor((H-1)/2), inclusive
    const int n_quads = (int) ((n_hi - n_lo) / 4) + 1;
    const int c2 = (int) (n_lo - in_lo) - (T - 1); // window start of quad 0 in the input buffer
    const int cj = (int) (2 * n_lo - L);           // local output index of quad 0's first value (0 or -1)
    const int NL = (int) (H - L);
    double fr[T];
#pragma unroll
    for (int j = 0; j < T; j++) fr[j] = f[j];
    // last stage: clip to the call's output range, in local coordinates
    int jl = 0, jh = NL;
    if (last) {
        if (p.e0 > L) jl = (int) (p.e0 - L);
        if (p.e1 < H) jh = (int) (p.e1 - L);
    }
    const bool neg = (L < 0); // stream values at negative indices are zeros, not filter outputs
    double* const obase = (last && dst.mask == -1) ? dst.ptr + (long long) ch * dst.stride + (L - dst.base) : nullptr;
    const bool vec_ok = obase != nullptr && ((reinterpret_cast<unsigned long long>(obase) & 15) == 0) && cj == 0;
    for (int q = tid; q < n_quads; q += HB_NT) {
        double w[2 * T + 3];
#pragma unroll
        for (int i = 0; i < 2 * T + 3; i++) {
            const int o = c2 + i;
            w[i] = in[5 * q + o + (o >> 2)];
        }
        double v[8];
#pragma unroll
        for (int m = 0; m < 4; m++) {
            double od = fr[0] * (w[T + m] + w[T - 1 + m]);
#pragma unroll
            for (int j = 1; j < T; j++) od = fma(fr[j], w[T + m + j] + w[T - 1 + m - j], od);
            v[2 * m] = w[T - 1 + m];
            v[2 * m + 1] = od;
        }
        const int j0 = 8 * q + cj;
        if (last) {
            if (vec_ok && j0 >= jl && j0 + 8 <= jh) {
#pragma unroll
                for (int m = 0; m < 4; m++)
                    *reinterpret_cast<double2*>(obase + j0 + 2 * m) = make_double2(v[2 * m], v[2 * m + 1]);
            } else if (obase != nullptr) {
#pragma unroll
                for (int m = 0; m < 8; m++)
                    if (j0 + m >= jl && j0 + m < jh) obase[j0 + m] = v[m];
            } else {
#pragma unroll
                for (int m = 0; m < 8; m++)
                    if (j0 + m >= jl && j0 + m < jh) dst_write(dst, ch, L + j0 + m, v[m]);
            }
        } else if (!neg && j0 >= 0 && j0 + 8 <= NL) {
#pragma unroll
            for (int m = 0; m < 8; m++) out[hb_lay(j0 + m, osh)] = v[m];
        } else {
#pragma unroll
            for (int m = 0; m < 8; m++)
                if (j0 + m >= 0 && j0 + m < NL) out[hb_lay(j0 + m, osh)] = (L + j0 + m < 0) ? 0.0 : v[m];
        }
    }
}

// The last two stages of the cascade in one pass (r8b_hbfuse.cuh): reads s_{c-2} from shared memory, writes s_c to
// global memory; s_{c-1} exists only in registers.  L, H: the tile's range of s_c (L >= 0, multiple of 8 apart).
template <int T1, int T2>
__device__ __forceinline__ void hb_stage_last2(const double* __restrict__ in, long long in_lo, const double* __restrict__ f1,
                                               const double* __restrict__ f2, long long L, long long H, int ish,
                                               const HbCascadeParams& p, const DstView& dst, int ch, int tid)
{
    using G = HbFuseGeom<T1, T2>;
    const long long n_lo = L >> 1;                 // first s_{c-1} position of the tile (even: L is a multiple of 4)
    const int n_items = (int) ((H - L) >> 3);      // 8 outputs each
    const int base = (int) ((n_lo >> 1) + G::UB - in_lo); // buffer-local index of item 0's first u sample
    const bool neg = n_lo - T2 + 1 < 0;            // only the very first tile of a stream
    double fr[T1], gr[T2];
#pragma unroll
    for (int j = 0; j < T1; j++) fr[j] = f1[j];
#pragma unroll
    for (int j = 0; j < T2; j++) gr[j] = f2[j];
    const int NL = (int) (H - L);
    int jl = 0, jh = NL; // clip to the call's output range, in tile-local coordinates
    if (p.e0 > L) jl = (int) (p.e0 - L);
    if (p.e1 < H) jh = (int) (p.e1 - L);
    double* const obase = (dst.mask == -1) ? dst.ptr + (long long) ch * dst.stride + (L - dst.base) : nullptr;
    const bool vec_ok = obase != nullptr && ((reinterpret_cast<unsigned long long>(obase) & 15) == 0);
    for (int q = tid; q < n_items; q += HB_NT) {
        const int o0 = base + 2 * q;
        double y8[8];
        hb_fused_item<T1, T2>(fr, gr, [&](int s) { return in[hb_lay(o0 + s, ish)]; }, n_lo + 4LL * q, neg, y8);
        const int j0 = 8 * q;
        if (vec_ok && j0 >= jl && j0 + 8 <= jh) {
#pragma unroll
            for (int m = 0; m < 4; m++)
                *reinterpret_cast<double2*>(obase + j0 + 2 * m) = make_double2(y8[2 * m], y8[2 * m + 1]);
        } else if (obase != nullptr) {
#pragma unroll
            for (int m = 0; m < 8; m++)
                if (j0 + m >= jl && j0 + m < jh) obase[j0 + m] = y8[m];
        } else {
#pragma unroll
            for (int m = 0; m < 8; m++)
                if (j0 + m >= jl && j0 + m < jh) dst_write(dst, ch, L + j0 + m, y8[m]);
        }
    }
}

// (T1, T2) pairs the fused last-two-stages pass is instantiated for.
bool hb_last2_supported(int t1, int t2) { return t1 >= 1 && t1 <= 6 && t2 >= 1 && t2 <= 4; }

int hbup_cascade_plan(HbCascadeParams& p, int smem_budget_doubles, bool allow_last2)
{
    const int cl = p.n_stages;
    // halos, from the last stage backwards (see k_hbup_cascade)
    p.lo_off[cl] = 0;
    p.hi_off[cl] = 0;
    for (int k = cl - 1; k >= 0; k--) {
        const int T = p.ntaps[k];
        p.lo_off[k] = (p.lo_off[k + 1] + 1) / 2 + T - 1;
        p.hi_off[k] = (p.hi_off[k + 1] >= 1 ? (p.hi_off[k + 1] - 1) / 2 : -1) + T + 1;
    }
    p.fuse_last2 = (cl >= 2 && allow_last2 && hb_last2_supported(p.ntaps[cl - 2], p.ntaps[cl - 1])) ? 1 : 0;
    const int nbuf = p.fuse_last2 ? cl - 1 : cl; // streams 0 .. nbuf-1 live in shared memory
    int halo = 0;
    for (int k = 0; k < nbuf; k++) halo += p.lo_off[k] + p.hi_off[k] + 8;
    // buffers carry a 5/4 skew
    int w = (((smem_budget_doubles * 4) / 5 - halo) / ((1 << nbuf) - 1)) & ~31;
    if (w > 1024) w = 1024;
    if (w < 32) w = 32;
    p.w = w;
    int off = 0;
    for (int k = 0; k < nbuf; k++) {
        p.boff[k] = off; // buffer k starts at its own lo bound
        off += (((w << k) + p.lo_off[k] + p.hi_off[k] + 8) * 5 + 3) / 4 + 2; // + slack: threads work in quads; 5/4 skew
        off = (off + 1) & ~1;
    }
    return off * (int) sizeof(double);
}

template <int T1>
__device__ __forceinline__ void hb_last2_dispatch(int t2, const double* in, long long in_lo, const double* f1, const double* f2,
                                                  long long L, long long H, int ish, const HbCascadeParams& p, const DstView& dst,
                                                  int ch, int tid)
{
    switch (t2) {
    case 1: hb_stage_last2<T1, 1>(in, in_lo, f1, f2, L, H, ish, p, dst, ch, tid); break;
    case 2: hb_stage_last2<T1, 2>(in, in_lo, f1, f2, L, H, ish, p, dst, ch, tid); break;
    case 3: hb_stage_last2<T1, 3>(in, in_lo, f1, f2, L, H, ish, p, dst, ch, tid); break;
    default: hb_stage_last2<T1, 4>(in, in_lo, f1, f2, L, H, ish, p, dst, ch, tid); break;
    }
}

// CTA shape of the cascade.  The kernel is bound by the block-wide barriers between its stage passes, not by a pipe, so
// more, smaller CTAs per SM overlap better: 4 x 128 threads with ~55 KB tiles measured 1.33 ms on cfg 4 against 1.45 ms
// for 2 x 256 threads with ~110 KB tiles (124 registers either way, no spills; 384 / 512 threads were slower still).
#ifndef R8BGPU_HB_MINB
#define R8BGPU_HB_MINB 4
#endif
__global__ void __launch_bounds__(HB_NT, R8BGPU_HB_MINB) k_hbup_cascade(HbCascadeParams p, SrcView src, DstView dst)
{
    extern __shared__ double hsm[];
    const int tid = threadIdx.x;
    const int ch = blockIdx.y;
    const long long A = p.a0 + (long long) blockIdx.x * p.w; // tile = s0 positions [A, A + w)
    const int c = p.n_stages;
    // layout shift of stream buffer k: the one the fused last-two-stages pass reads is laid out for its 2-sample lane stride
    auto sh_of = [&](int k) { return (p.fuse_last2 && k == c - 2) ? 4 : 2; };

    // stage 0: gather the input segment
    {
        const long long lo = A - p.lo_off[0], hi = A + p.w + p.hi_off[0];
        double* b0 = hsm + p.boff[0];
        for (long long n = lo + tid; n < hi; n += HB_NT) b0[hb_lay((int) (n - lo), sh_of(0))] = (n < 0) ? 0.0 : src_read(src, ch, n);
    }
    __syncthreads();
#pragma unroll 1
    for (int k = 0; k < c; k++) {
        const double* __restrict__ in = hsm + p.boff[k];
        const long long in_lo = (A << k) - p.lo_off[k];
        if (p.fuse_last2 && k + 2 == c) { // stages c-2 and c-1 in one pass; s_{c-1} never reaches shared memory
            const long long L2 = A << c, H2 = (A + p.w) << c;
            const double* f1 = p.taps[k];
            const double* f2 = p.taps[k + 1];
            switch (p.ntaps[k]) {
            case 1: hb_last2_dispatch<1>(p.ntaps[k + 1], in, in_lo, f1, f2, L2, H2, sh_of(k), p, dst, ch, tid); break;
            case 2: hb_last2_dispatch<2>(p.ntaps[k + 1], in, in_lo, f1, f2, L2, H2, sh_of(k), p, dst, ch, tid); break;
            case 3: hb_last2_dispatch<3>(p.ntaps[k + 1], in, in_lo, f1, f2, L2, H2, sh_of(k), p, dst, ch, tid); break;
            case 4: hb_last2_dispatch<4>(p.ntaps[k + 1], in, in_lo, f1, f2, L2, H2, sh_of(k), p, dst, ch, tid); break;
            case 5: hb_last2_dispatch<5>(p.ntaps[k + 1], in, in_lo, f1, f2, L2, H2, sh_of(k), p, dst, ch, tid); break;
            default: hb_last2_dispatch<6>(p.ntaps[k + 1], in, in_lo, f1, f2, L2, H2, sh_of(k), p, dst, ch, tid); break;
            }
            break;
        }
        const bool last = (k + 1 == c);
        const long long L = last ? (A << c) : ((A << (k + 1)) - p.lo_off[k + 1]);
        const long long H = last ? ((A + p.w) << c) : (((A + p.w) << (k + 1)) + p.hi_off[k + 1]);
        double* out = last ? nullptr : hsm + p.boff[k + 1];
        const double* __restrict__ f = p.taps[k];
        switch (p.ntaps[k]) {
        case 1: hb_stage<1>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 2: hb_stage<2>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 3: hb_stage<3>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 4: hb_stage<4>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 5: hb_stage<5>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 6: hb_stage<6>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 7: hb_stage<7>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 8: hb_stage<8>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 9: hb_stage<9>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 10: hb_stage<10>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 11: hb_stage<11>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 12: hb_stage<12>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        case 13: hb_stage<13>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        default: hb_stage<14>(in, in_lo, f, L, H, out, last, sh_of(k + 1), p, dst, ch, tid); break;
        }
        __syncthreads();
    }
}

void launch_hbup_cascade(const HbCascadeParams& p, int smem_bytes, const SrcView& src, const DstView& dst,
                         int n_ch, cudaStream_t st)
{
    if (p.n_tiles <= 0 || n_ch <= 0) return;
    ensure_dyn_smem<k_hbup_cascade>(220 * 1024);
    dim3 grid((unsigned) p.n_tiles, (unsigned) n_ch);
    k_hbup_cascade<<<grid, HB_NT, smem_bytes, st>>>(p, src, dst);
}

namespace {
__global__ void __launch_bounds__(1024) k_dfma_peak(double* out, int iters, double a, double b)
{
    double acc[16];
#pragma unroll
    for (int i = 0; i < 16; i++) acc[i] = threadIdx.x * 1e-3 + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 16; i++) acc[i] = fma(acc[i], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 16; i++) s += acc[i];
    if (s == 12345.678) out[0] = s; // never true: keeps the chains alive without a store stream
}
} // namespace

double measure_dfma_tflops()
{
    int dev = 0, n_sm = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1.0;
    if (cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1.0;
    double* out = nullptr;
    if (cudaMalloc(&out, sizeof(double)) != cudaSuccess) return -1.0;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    const int iters = 8192, nt = 1024;
    double best = -1.0;
    for (int rep = 0; rep < 4; rep++) {
        cudaEventRecord(e0, 0);
        k_dfma_peak<<<n_sm, nt>>>(out, iters, 1.0000001, 1e-9);
        cudaEventRecord(e1, 0);
        if (cudaEventSynchronize(e1) != cudaSuccess) break;
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        const double tf = 2.0 * 16.0 * iters * (double) nt * n_sm / (ms * 1e-3) / 1e12;
        if (rep > 0 && tf > best) best = tf; // first launch is the warm-up
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(out);
    return best;
}

} // namespace r8bgpu

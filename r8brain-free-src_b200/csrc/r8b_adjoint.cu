// r8b_adjoint.cu -- transposed stage operators: gradients through whole-clip resampling (r8bgpu_batch_oneshot_adjoint).
//
// Every kernel computes the gradient of one stage's INPUT stream from the gradient of its OUTPUT stream, for all clips of
// the call at once (one 1-D grid over the clips' tiles).  Each input-gradient sample is a gather: one thread sums, in ascending output
// order, the terms of the outputs that read it.  No atomics, so the bytes do not depend on the launch geometry.
//
//   k_bc_adj         BlockConv (U, D), taps h[-L..L]:  x[n] = sum_q h[D q - U n] g[q]
//   k_bcx_adj        block-exact BlockConv: block b's contribution c_b[m] = sum_{q in b} K(n_q, m) g[q] over its window
//   k_bcx_sum        x[n] = sum over the blocks whose window covers U n of c_b, in block order
//   k_frac_adj<P>    interpolators: x[n] = sum over outputs j whose window covers n of c_j[n - p_j + fll] g[j]
//   k_crop_accum     crops: each clip's input gradient, the sum of its crops' rows in crop order
// The half-band stages run on k_hbdown / k_hbup with the other direction's taps (DESIGN.md K9).  Indices are absolute;
// each row starts at its window's origin (AdjClip), and the sums run over the g window only.
#include "r8b_kernels.h"

namespace r8bgpu {

namespace {

__device__ __forceinline__ long long floor_div(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// read position and fraction (order 2) or phase (whole stepping) of output j -- k_frac's frac_position on the call record
// that holds j; r: a record index at or below j's (advanced in place)
template <bool POLY>
__device__ __forceinline__ long long adj_pos(const AdjParams& p, const AdjPolyRec* __restrict__ rec, int nrec, int& r,
                                             long long j, double& fpos, int& phase)
{
    if constexpr (!POLY) {
        const long long pos = j * p.in_step;
        const long long ip = pos / p.out_step;
        phase = (int) (pos - ip * p.out_step);
        fpos = 0.0;
        return ip;
    } else {
        while (r + 1 < nrec && rec[r + 1].e0 <= j) r++;
        const AdjPolyRec& c = rec[r];
        const long long k = j - c.e0;
        phase = 0;
        if (k == 0) {
            fpos = c.fpos0;
            return c.p0;
        }
        const int ic = c.in_counter0 + (int) k;
        const double np = __ddiv_rn(__dmul_rn(__dadd_rn((double) ic, c.in_pos_shift), c.ssr), c.dsr);
        const int ni = __double2int_rz(np);
        fpos = __dsub_rn(np, (double) ni);
        return c.p0 + (ni - c.in_pos_int0);
    }
}

// the record holding output j (records are sorted by e0 and cover [0, ng))
__device__ __forceinline__ int adj_rec_of(const AdjPolyRec* __restrict__ rec, int nrec, long long j)
{
    int lo = 0, hi = nrec - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (rec[mid].e0 <= j) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

} // namespace

// Work units of 256 threads, clip-major: `per` units per clip.  One 1-D grid strides over all of them, so neither the
// clip count nor a stage's block count meets the 65535 limit of gridDim.y / gridDim.z.
constexpr long long ADJ_MAX_CTAS = 1LL << 20;

__device__ __forceinline__ void bc_adj_sample(const AdjParams& p, int r, long long n)
{
    const AdjClip c = p.clip[r];
    n += c.x0;
    if (n >= c.nx) return;
    const double* __restrict__ g = p.g + (long long) r * p.g_stride - c.g0;
    const long long un = (long long) p.U * n;
    long long q0 = -floor_div(-(un - p.L), p.D), q1 = floor_div(un + p.L, p.D);
    if (q0 < c.g0) q0 = c.g0;
    if (q1 > c.ng - 1) q1 = c.ng - 1;
    double acc = 0.0;
    for (long long q = q0; q <= q1; q++) acc = fma(__ldg(p.h + (p.D * q - un + p.L)), __ldg(g + q), acc);
    p.x[(long long) r * p.x_stride + (n - c.x0)] = acc;
}

__global__ void __launch_bounds__(256) k_bc_adj(const __grid_constant__ AdjParams p, long long per, long long units)
{
    for (long long u = blockIdx.x; u < units; u += gridDim.x) {
        const int r = (int) (u / per);
        bc_adj_sample(p, r, (u - r * per) * 256 + threadIdx.x);
    }
}

// Block b's window is the tile stream's [b il - prev, b il - prev + M); its outputs q have D q in [b il - L, (b+1) il - L).
// Output q reads window sample m with weight kappa[(n_q - m) mod M] + nyq (-1)^(n_q / D) u[m], n_q = D q - (b il - prev).
__device__ __forceinline__ void bcx_adj_sample(const AdjParams& p, int r, long long b, int m)
{
    const AdjClip c = p.clip[r];
    b += c.b0;
    if (b >= c.nb || m >= p.M) return;
    const double* __restrict__ g = p.g + (long long) r * p.g_stride - c.g0;
    const long long start = b * p.il - p.prev;
    long long q0 = -floor_div(-(b * p.il - p.L), p.D), q1 = -floor_div(-((b + 1) * p.il - p.L), p.D) - 1;
    if (q0 < c.g0) q0 = c.g0;
    if (q1 > c.ng - 1) q1 = c.ng - 1;
    double acc = 0.0, nq_acc = 0.0;
    for (long long q = q0; q <= q1; q++) {
        const long long nq = p.D * q - start;
        const double gq = __ldg(g + q);
        acc = fma(__ldg(p.kappa + ((nq - m) & (p.M - 1))), gq, acc);
        nq_acc += ((nq / p.D) & 1) ? -gq : gq;
    }
    p.contrib[(long long) r * p.c_stride + (b - c.b0) * p.M + m] = fma(p.nyq * nq_acc, __ldg(p.u + m), acc);
}

// units: clip-major, then block, then 256-sample pieces of the window (mt per block)
__global__ void __launch_bounds__(256) k_bcx_adj(const __grid_constant__ AdjParams p, long long nb, int mt, long long units)
{
    for (long long u = blockIdx.x; u < units; u += gridDim.x) {
        const long long per = nb * mt;
        const int r = (int) (u / per);
        const long long v = u - r * per, b = v / mt;
        bcx_adj_sample(p, r, b, (int) (v - b * mt) * 256 + threadIdx.x);
    }
}

__device__ __forceinline__ void bcx_sum_sample(const AdjParams& p, int r, long long n)
{
    const AdjClip c = p.clip[r];
    n += c.x0;
    if (n >= c.nx) return;
    const double* __restrict__ cb = p.contrib + (long long) r * p.c_stride - c.b0 * p.M;
    const long long t = (long long) p.U * n;
    long long b0 = -floor_div(-(t - p.M + 1 + p.prev), p.il), b1 = floor_div(t + p.prev, p.il);
    if (b0 < c.b0) b0 = c.b0;
    if (b1 > c.nb - 1) b1 = c.nb - 1;
    double acc = 0.0;
    for (long long b = b0; b <= b1; b++) acc += __ldg(cb + b * p.M + (t - (b * p.il - p.prev)));
    p.x[(long long) r * p.x_stride + (n - c.x0)] = acc;
}

__global__ void __launch_bounds__(256) k_bcx_sum(const __grid_constant__ AdjParams p, long long per, long long units)
{
    for (long long u = blockIdx.x; u < units; u += gridDim.x) {
        const int r = (int) (u / per);
        bcx_sum_sample(p, r, (u - r * per) * 256 + threadIdx.x);
    }
}

template <bool POLY>
__device__ __forceinline__ void frac_adj_sample(const AdjParams& p, int r, long long n)
{
    const AdjClip c = p.clip[r];
    n += c.x0;
    if (n >= c.nx) return;
    const double* __restrict__ g = p.g + (long long) r * p.g_stride - c.g0;
    const AdjPolyRec* __restrict__ rec = POLY ? p.rec + c.rec0 : nullptr;
    const int nrec = c.nrec;
    double acc = 0.0;
    if (c.ng > c.g0 && (!POLY || nrec > 0)) {
        // output j reads [p_j - fll, p_j - fll + flen): n is read by the outputs with p_j in [n + fll - flen + 1, n + fll]
        const long long lo_p = n + p.fll - p.flen + 1, hi_p = n + p.fll;
        double fp;
        int ph, ri = 0;
        long long lo = c.g0, hi = c.ng; // first j with p_j >= lo_p
        while (lo < hi) {
            const long long mid = lo + (hi - lo) / 2;
            if (POLY) ri = adj_rec_of(rec, nrec, mid);
            if (adj_pos<POLY>(p, rec, nrec, ri, mid, fp, ph) >= lo_p) hi = mid;
            else lo = mid + 1;
        }
        if (POLY && lo < c.ng) ri = adj_rec_of(rec, nrec, lo);
        for (long long j = lo; j < c.ng; j++) {
            const long long ip = adj_pos<POLY>(p, rec, nrec, ri, j, fp, ph);
            if (ip > hi_p) break;
            const int i = (int) (n - ip + p.fll);
            double coef;
            if (!POLY) {
                coef = __ldg(p.bank + (long long) ph * p.flen + i);
            } else {
                double x = __dmul_rn(fp, (double) p.fracs);
                const int fti = __double2int_rz(x);
                x = __dsub_rn(x, (double) fti);
                const double x2 = __dmul_rn(x, x);
                const double* row = p.bank + (long long) fti * p.flen * 3 + 3 * i;
                coef = fma(__ldg(row + 2), x2, fma(__ldg(row + 1), x, __ldg(row)));
            }
            acc = fma(coef, __ldg(g + j), acc);
        }
    }
    p.x[(long long) r * p.x_stride + (n - c.x0)] = acc;
}

template <bool POLY>
__global__ void __launch_bounds__(256) k_frac_adj(const __grid_constant__ AdjParams p, long long per, long long units)
{
    for (long long u = blockIdx.x; u < units; u += gridDim.x) {
        const int r = (int) (u / per);
        frac_adj_sample<POLY>(p, r, (u - r * per) * 256 + threadIdx.x);
    }
}

// One thread per (clip, hull sample): the clip's crop rows that cover the sample, summed in ascending crop order.
__global__ void __launch_bounds__(256) k_crop_accum(const __grid_constant__ CropAccParams p, long long per, long long units)
{
    for (long long u = blockIdx.x; u < units; u += gridDim.x) {
        const int r = (int) (u / per);
        const CropAccClip c = p.clips[r];
        const long long n = c.lo + (u - r * per) * 256 + threadIdx.x;
        if (n >= c.hi) continue;
        double acc = 0.0;
        bool any = false;
        for (int k = c.k0; k < c.k0 + c.nk; k++) {
            const CropAccRow w = p.rows[k];
            if (n < w.x0 || n >= w.x1) continue;
            const double v = __ldg(p.x + w.row * p.x_stride + (n - w.x0));
            acc = any ? acc + v : v;
            any = true;
        }
        const long long at = p.interleaved ? n * p.out_stride + c.out : c.out * p.out_stride + n;
        if (p.fmt == FMT_F64) static_cast<double*>(p.out)[at] = acc;
        else static_cast<float*>(p.out)[at] = (float) acc;
    }
}

static unsigned adj_grid(long long units) { return (unsigned) (units < ADJ_MAX_CTAS ? units : ADJ_MAX_CTAS); }

void launch_bc_adj(const AdjParams& p, long long max_nx, int n_clips, cudaStream_t st)
{
    if (max_nx <= 0 || n_clips <= 0) return;
    const long long per = (max_nx + 255) / 256, units = per * n_clips;
    k_bc_adj<<<adj_grid(units), 256, 0, st>>>(p, per, units);
}

void launch_bcx_adj(const AdjParams& p, long long max_nb, long long max_nx, int n_clips, cudaStream_t st)
{
    if (n_clips <= 0) return;
    if (max_nb > 0) {
        const int mt = (p.M + 255) / 256;
        const long long units = max_nb * mt * n_clips;
        k_bcx_adj<<<adj_grid(units), 256, 0, st>>>(p, max_nb, mt, units);
    }
    if (max_nx > 0) {
        const long long per = (max_nx + 255) / 256, units = per * n_clips;
        k_bcx_sum<<<adj_grid(units), 256, 0, st>>>(p, per, units);
    }
}

void launch_frac_adj(const AdjParams& p, bool poly, long long max_nx, int n_clips, cudaStream_t st)
{
    if (max_nx <= 0 || n_clips <= 0) return;
    const long long per = (max_nx + 255) / 256, units = per * n_clips;
    if (poly) k_frac_adj<true><<<adj_grid(units), 256, 0, st>>>(p, per, units);
    else k_frac_adj<false><<<adj_grid(units), 256, 0, st>>>(p, per, units);
}

void launch_crop_accum(const CropAccParams& p, long long max_hull, int n_clips, cudaStream_t st)
{
    if (max_hull <= 0 || n_clips <= 0) return;
    const long long per = (max_hull + 255) / 256, units = per * n_clips;
    k_crop_accum<<<adj_grid(units), 256, 0, st>>>(p, per, units);
}

} // namespace r8bgpu

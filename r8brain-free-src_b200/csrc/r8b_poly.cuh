// r8b_poly.cuh -- timing arithmetic of the order-2 (non-whole-stepping) interpolator shared by the two fused kernels
// (CDSPFracInterpolator::convolve2, CDSPFracInterpolator.h:1069-1179): where output k of a call reads the stream.
#pragma once
#include <cuda_runtime.h>

#include <cmath>

#include "r8b_fft.cuh"
#include "r8b_fused_common.cuh"
#include "r8b_kernels.h"

namespace r8bgpu {

// Position and fraction of output k of this call; the reference's IEEE expression order
// ((InCounter + InPosShift) * ssr) / dsr (CDSPFracInterpolator.h:1161-1166), or the host-walked
// R8B_FASTTIMING sequence.  Also compiles for the host (the v2 kernel's tile table, r8b_fused2_core.cuh), where the
// same IEEE operations are plain expressions (built without floating-point contraction).
R8B_HD void poly_position(const FusedParams& p, long long k, long long& ip, double& fpos)
{
    ip = p.p0;
    fpos = p.fpos0;
    if (p.pos_dp != nullptr) {
        ip = p.p0 + R8B_LDG(p.pos_dp + k);
        fpos = R8B_LDG(p.pos_fpos + k);
    } else if (k > 0) {
        const int ic = p.in_counter0 + (int) k;
#ifdef __CUDA_ARCH__
        const double np = __ddiv_rn(__dmul_rn(__dadd_rn((double) ic, p.in_pos_shift), p.ssr), p.dsr);
        const int ni = __double2int_rz(np);
        ip = p.p0 + (ni - p.in_pos_int0);
        fpos = __dsub_rn(np, (double) ni);
#else
        const double np = (((double) ic + p.in_pos_shift) * p.ssr) / p.dsr;
        const int ni = (int) np;
        ip = p.p0 + (ni - p.in_pos_int0);
        fpos = np - (double) ni;
#endif
    }
}

// First k in [0, nk] whose position is >= lim (positions are non-decreasing in k).
R8B_HD long long poly_first_k(const FusedParams& p, long long lim, long long nk)
{
    auto pos = [&](long long k) {
        long long ip;
        double f;
        poly_position(p, k, ip, f);
        return ip;
    };
    if (p.pos_dp != nullptr) { // table: binary search
        long long lo = 0, hi = nk;
        while (lo < hi) {
            const long long mid = lo + (hi - lo) / 2;
            if (pos(mid) >= lim) hi = mid;
            else lo = mid + 1;
        }
        return lo;
    }
    // closed form: invert the timing expression, then settle on the exact integer with the exact expression
    const double t = (double) (lim - p.p0 + p.in_pos_int0);
    double est = ceil(t * p.dsr / p.ssr - p.in_pos_shift - (double) p.in_counter0);
    long long k = est < 0.0 ? 0 : (est > (double) nk ? nk : (long long) est);
    while (k > 0 && pos(k - 1) >= lim) k--;
    while (k < nk && pos(k) < lim) k++;
    return k;
}

// ---- k_up2_frac's order-2 bookkeeping (r8b_fused.cu); also compiles for the host, where tests/cpp/order2_pairs.cpp
// replays it pair by pair ---------------------------------------------------------------------------------------------

constexpr int POLY_QUEUE = 1024; // deferred outputs per chunk (4 KB of dynamic shared memory behind the staged rows)

// Circular run of bank rows used by outputs [k_lo, k_hi): first row and number of rows to stage (0 = none).
// One row of margin on either side: rounding of the fraction may step past the end rows.  Rows outside the
// staged run are always read from global memory, so this is an optimisation only.
R8B_HD void poly_rows_for(const FusedParams& p, long long k_lo, long long k_hi, int& r_lo, int& n_st)
{
    r_lo = 0;
    n_st = 0;
    if (p.poly_dir == 0 || p.poly_rows_cap <= 0 || k_hi <= k_lo) return;
    long long ip;
    double f0, f1;
    poly_position(p, k_lo, ip, f0);
    poly_position(p, k_hi - 1, ip, f1);
#ifdef __CUDA_ARCH__
    int ra = __double2int_rz(__dmul_rn(f0, (double) p.fracs));
    int rb = __double2int_rz(__dmul_rn(f1, (double) p.fracs));
#else
    int ra = (int) (f0 * (double) p.fracs);
    int rb = (int) (f1 * (double) p.fracs);
#endif
    if (ra >= p.fracs) ra = p.fracs - 1;
    if (rb >= p.fracs) rb = p.fracs - 1;
    const int first = p.poly_dir > 0 ? ra : rb, last = p.poly_dir > 0 ? rb : ra;
    int cnt = last - first;
    if (cnt < 0) cnt += p.fracs;
    cnt += 3;
    r_lo = first > 0 ? first - 1 : p.fracs - 1;
    n_st = cnt < p.poly_rows_cap ? cnt : p.poly_rows_cap;
    if (n_st > p.fracs) n_st = p.fracs;
}

// Outputs [ka, kb) of a pair are processed in p.poly_chunks equal pieces, each with its own staged rows.
R8B_HD long long poly_chunk_start(long long ka, long long kb, int c, int n_chunks)
{
    return ka + (kb - ka) * c / n_chunks;
}

struct PolyOut {          // everything one output needs
    double x, x2;
    int fti, yi;          // bank row; logical index of the window start in its tile buffer
    bool use_b, ok;
};

// Output k of the call in a tile pair whose y buffers start at absolute 2x index ya0 (tile a) and yb0 (tile b), windows
// starting at or after bsel reading tile b: its bank row and fraction, and where its flen-sample window lies.  ok: the
// window lies inside its 2 * FM-sample tile buffer (always so for an output the pair owns).
R8B_HD PolyOut poly_output(const FusedParams& p, long long ya0, long long yb0, long long bsel, long long k)
{
    PolyOut o;
    long long ip;
    double fpos;
    poly_position(p, k, ip, fpos);
#ifdef __CUDA_ARCH__
    double x = __dmul_rn(fpos, (double) p.fracs);
    o.fti = __double2int_rz(x);
    x = __dsub_rn(x, (double) o.fti);
    o.x = x;
    o.x2 = __dmul_rn(x, x);
#else
    double x = fpos * (double) p.fracs;
    o.fti = (int) x;
    x = x - (double) o.fti;
    o.x = x;
    o.x2 = x * x;
#endif
    const long long ws = ip - p.fll;
    o.use_b = ws >= bsel;
    o.yi = (int) (ws - (o.use_b ? yb0 : ya0));
    o.ok = o.yi >= 0 && o.yi + p.flen <= 2 * FM; // always true for owned outputs
    return o;
}

// Slot of bank row fti in the staged run starting at row r_lo (a slot >= n_st: the row is not staged).
R8B_HD int poly_slot(const FusedParams& p, int r_lo, int fti)
{
    int slot = fti - r_lo;
    if (slot < 0) slot += p.fracs;
    return slot;
}

// Four consecutive outputs o[0..nv) of one thread share their coefficient loads (poly_block4<NN>) when all four are
// there, their windows lie in the same tile NN samples apart, and they read one staged bank row.
template <int NN>
R8B_HD bool poly_fast_group(const FusedParams& p, const PolyOut (&o)[4], int nv, int r_lo, int n_st, int& slot)
{
    bool fast = nv == 4 && o[0].ok && o[3].ok;
    if (fast) {
#pragma unroll
        for (int r = 1; r < 4; r++)
            fast = fast && o[r].fti == o[0].fti && o[r].use_b == o[0].use_b && o[r].yi == o[0].yi + NN * r;
    }
    slot = poly_slot(p, r_lo, o[0].fti);
    return fast && slot < n_st && o[0].fti < p.fracs;
}

} // namespace r8bgpu

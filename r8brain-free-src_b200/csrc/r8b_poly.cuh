// r8b_poly.cuh -- timing arithmetic of the order-2 (non-whole-stepping) interpolator shared by the two fused kernels
// (CDSPFracInterpolator::convolve2, CDSPFracInterpolator.h:1069-1179): where output k of a call reads the stream.
#pragma once
#include <cuda_runtime.h>

#include <cmath>

#include "r8b_fft.cuh"
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


} // namespace r8bgpu

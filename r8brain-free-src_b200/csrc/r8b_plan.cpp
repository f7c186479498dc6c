// r8b_plan.cpp -- see r8b_plan.h.  Strict-IEEE host code (build with -ffp-contract=off).
#include "r8b_plan.h"
#include "../../include/r8bgpu.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>

namespace r8bgpu {

namespace {

long long ceil_div(long long a, long long b) { return (a + b - 1) / b; } // a >= 0, b > 0

const char* const kStageNames[5] = {"BlockConv", "FracInterp whole-step", "FracInterp order-2", "HBUp", "HBDown"};

bool make_blockconv(StageDesc& s, double norm_freq, double tb, double atten, double gain, int up,
                    int down, int extfft, std::string& err)
{
    s.kind = ST_BLOCKCONV;
    s.up = up;
    s.down = down;
    s.norm_freq = norm_freq;
    s.trans_band = tb;
    s.gain = gain;
    if (!design_lowpass(norm_freq, tb, atten, gain, extfft, s.lp)) {
        err = "low-pass design parameters out of range";
        return false;
    }
    // Block geometry of the reference convolver -- needed only to reproduce WHEN samples are
    // emitted (CDSPBlockConvolver.h:75-146); the CUDA tiles use their own FFT size.
    const int K = s.lp.kernel_len, L = s.lp.half_len;
    const int b2 = 2 << s.lp.block_len_bits;
    int ushift = bit_occupancy(up) - 1;
    int prev_len, in_len;
    if ((1 << ushift) == up) {
        prev_len = (K - 1 + up - 1) / up;
        in_len = b2 - prev_len * up;
    } else {
        ushift = -1;
        prev_len = K - 1;
        in_len = b2 - prev_len;
    }
    int latency = in_len + L;
    const int dshift = bit_occupancy(down) - 1;
    if ((1 << dshift) == down && down > 1) {
        if (ushift > 0) {
            err = "power-of-two up- and down-factors together are not planned by the reference";
            return false;
        }
        const int ilc = in_len & (down - 1);
        prev_len += ilc;
        in_len -= ilc;
        latency -= ilc;
        s.block_exact = true;
    }
    s.ref_input_len = in_len;
    s.ref_prev_len = prev_len;
    s.latency = latency;
    const int lg = (L + up - 1) / up + 1;
    s.src_history = (latency + L + up - 1) / up + lg + 40;
    if (s.block_exact) s.src_history = 2 * b2 + 16;
    return true;
}

bool make_frac(StageDesc& s, double src, double dst, double atten, bool is_third, int fasttiming,
               std::string& err, bool no_whole = false)
{
    s.src_rate = src;
    s.dst_rate = dst;
    s.is_third = is_third;
    int a = 0, b = 0;
    if (!no_whole && whole_stepping(src, dst, a, b)) {
        s.kind = ST_FRAC_WHOLE;
        s.in_step = a;
        s.out_step = b;
        design_frac_bank(b, atten, is_third, s.bank);
    } else {
        s.fasttiming = fasttiming != 0;
        s.kind = ST_FRAC_POLY;
        design_frac_bank(-1, atten, is_third, s.bank);
    }
    s.src_history = s.bank.filter_len + 8;
    return true;
}

void make_hb(StageDesc& s, StageKind kind, double atten, int steep, bool is_third)
{
    s.kind = kind;
    s.steep_index = steep;
    s.is_third = is_third;
    const HalfbandTaps t = select_halfband(atten, steep, is_third);
    s.hb_taps = t.ntaps;
    s.hb_atten = t.atten;
    s.hb.assign(t.taps, t.taps + t.ntaps);
    s.src_history = (kind == ST_HBUP ? 2 : 4) * t.ntaps + 8;
}

// The reference computes this chain in int (getMaxOutLen); here it is 64-bit, so that a chain past R8BGPU_MAX_LEN is
// refused instead of wrapping.  max_in <= R8BGPU_MAX_LEN and every stage ratio is small, so nothing here overflows.
long long stage_max_out_len(const StageDesc& s, long long max_in)
{
    switch (s.kind) {
    case ST_BLOCKCONV:
        return (max_in * s.up + s.down - 1) / s.down;                    // CDSPBlockConvolver.h:208-213
    case ST_FRAC_WHOLE:
    case ST_FRAC_POLY:
        return (long long) std::ceil(max_in * s.dst_rate / s.src_rate) + 1; // CDSPFracInterpolator.h:827-832
    case ST_HBUP:
        return max_in * 2;                                                 // CDSPHBUpsampler.h:648-653
    case ST_HBDOWN:
        return (max_in + 1) >> 1;                                          // CDSPHBDownsampler.h:113-118
    }
    return 0;
}

// Stores stage i's buffer length, or refuses it (false, with err) when it exceeds R8BGPU_MAX_LEN.
bool set_max_out_len(StageDesc& s, size_t i, long long len, std::string& err)
{
    if (len > R8BGPU_MAX_LEN) {
        err = "stage " + std::to_string(i) + " (" + kStageNames[s.kind] + ") would need max_out_len " + std::to_string(len) +
              ", above R8BGPU_MAX_LEN = " + std::to_string(R8BGPU_MAX_LEN) + "; use a smaller MaxInLen";
        return false;
    }
    s.max_out_len = (int) len;
    return true;
}

int stage_in_len_before_out_pos(const StageDesc& s, int pos)
{
    switch (s.kind) {
    case ST_BLOCKCONV: // CDSPBlockConvolver.h:192-196 (LatencyFrac == 0 for linear phase)
        return (int) ((s.latency + (double) pos * s.down) / s.up + 0.0 * s.down / s.up);
    case ST_FRAC_WHOLE: // CDSPFracInterpolator.h:802-811
        return s.bank.filter_len / 2 +
            (int) ((0 + (double) pos * s.in_step) / s.out_step + 0.0 * s.in_step / s.out_step);
    case ST_FRAC_POLY: // :813-814
        return s.bank.filter_len / 2 + (int) (0.0 + pos * s.src_rate / s.dst_rate);
    case ST_HBUP: // CDSPHBUpsampler.h:633-636
        return s.hb_taps + (int) ((0 + 0.0 + pos) * 0.5);
    case ST_HBDOWN: // CDSPHBDownsampler.h:98-101
        return (2 * s.hb_taps - 1) + (int) ((0 + 0.0 + pos) * 2.0);
    }
    return 0;
}

} // namespace

long long blockconv_emitted(const StageDesc& s, long long n)
{
    const long long avail = (long long) s.up * n - s.latency;
    return avail <= 0 ? 0 : ceil_div(avail, s.down);
}

long long frac_whole_emitted(const StageDesc& s, long long n)
{
    // outputs j >= 0 with floor(j*InStep/OutStep) + fl2 <= n-1
    const long long fl2 = s.bank.filter_len / 2;
    const long long pmax = n - 1 - fl2;
    if (pmax < 0) return 0;
    // floor(j*a/b) <= pmax  <=>  j*a <= pmax*b + b - 1  <=>  j <= (pmax*b + b - 1)/a
    const long long a = s.in_step, b = s.out_step;
    return (pmax * b + b - 1) / a + 1;
}

long long hbup_emitted(const StageDesc& s, long long n)
{
    const long long c = n - s.hb_taps;
    return c <= 0 ? 0 : 2 * c;
}

long long hbdown_emitted(const StageDesc& s, long long n)
{
    const long long c = n / 2 - (s.hb_taps - 1);
    return c <= 0 ? 0 : c;
}

bool Plan::build(double src, double dst, int max_in, double tb, double att, int phase, int ext,
                 int fasttiming, bool no_whole, bool force_interp)
{
    src_rate = src;
    dst_rate = dst;
    max_in_len = max_in;
    trans_band = tb;
    atten = att;
    extfft = ext ? 1 : 0;
    this->fasttiming = fasttiming ? 1 : 0;
    stages.clear();
    passthrough = false;
    error.clear();
    max_out_len = max_in;
    max_trim = 0.0;
    trim_stage = -1;

    if (!(src > 0.0) || !(dst > 0.0) || max_in <= 0) {
        error = "invalid sample rates or MaxInLen";
        return false;
    }
    if (max_in > R8BGPU_MAX_LEN) {
        error = "MaxInLen " + std::to_string(max_in) + " is above R8BGPU_MAX_LEN = " + std::to_string(R8BGPU_MAX_LEN);
        return false;
    }
    if (phase != 0) {
        error = "only fprLinearPhase is implemented (minimum-phase is out of scope)";
        return false;
    }
    // force_interp skips exactly the constructor's shortcuts that end the chain without an interpolator: this return,
    // the single-step ratios (1), whole 2^c / 3*2^c upsampling (2) and the exact 2x / 3x decimation in (4).  Every other
    // decision, the whole-stepping preference in (3) included, stays the constructor's.
    if (src == dst && !force_interp) { // CDSPResampler.h:135-138
        passthrough = true;
        return true;
    }

    auto push_bc = [&](double nf, double tbw, double gain, int up, int down) -> bool {
        StageDesc s;
        if (!make_blockconv(s, nf, tbw, att, gain, up, down, extfft, error)) return false;
        stages.push_back(std::move(s));
        return true;
    };
    auto push_frac = [&](double s_rate, double d_rate, bool third) -> bool {
        StageDesc s;
        if (!make_frac(s, s_rate, d_rate, att, third, fasttiming, error, no_whole)) return false;
        stages.push_back(std::move(s));
        return true;
    };
    auto push_hb = [&](StageKind k, int steep, bool third) {
        StageDesc s;
        make_hb(s, k, att, steep, third);
        stages.push_back(std::move(s));
    };

    bool done = false;

    // (1) single-step common ratios, CDSPResampler.h:146-172
    static const int kCommon[5][2] = {{1, 2}, {1, 3}, {2, 3}, {3, 2}, {3, 4}};
    for (int i = 0; i < 5 && !done && !force_interp; i++) {
        const int num = kCommon[i][0], den = kCommon[i][1];
        if (src * num == dst * den) {
            if (!push_bc(1.0 / (num > den ? num : den), tb, num, num, den)) return false;
            done = true;
        }
    }

    // (2) whole 2^c or 3*2^c upsampling, :176-216
    for (int i = 2; i <= 3 && !done && !force_interp; i++) {
        bool found = false;
        int c = 0;
        while (true) {
            const double nsr = src * (i << c);
            if (nsr == dst) {
                found = true;
                break;
            }
            if (nsr > dst) break;
            c++;
        }
        if (found) {
            if (!push_bc(1.0 / i, tb, i, i, 1)) return false;
            for (int k = 0; k < c; k++) push_hb(ST_HBUP, k, i == 3);
            done = true;
        }
    }

    if (!done && dst * 2.0 > src) {
        // (3) upsampling or fractional downsampling down to 2X, :218-333
        const double nf = (dst > src ? 0.5 : 0.5 * dst / src);
        if (!push_bc(nf, tb, 2.0, 2, 1)) return false;

        const double tbw = 0.0175;
        const double thresh = src / (1.0 - tbw * tb);
        int c = 0, div = 1;
        while (true) {
            const int ndiv = div * 2;
            if (dst < thresh * ndiv) break;
            div = ndiv;
            c++;
        }
        int c2 = 0, div2 = 1;
        while (true) {
            const int ndiv = div * (c2 == 0 ? 3 : 2);
            if (dst < thresh * ndiv) break;
            div2 = ndiv;
            c2++;
        }
        const double src2 = src * 2.0;
        int t1, t2;
        if (c == 1 && whole_stepping(src2, dst, t1, t2)) c = 0;

        if (c > 0) {
            int num;
            if (c2 > 0 && div2 > div) {
                div = div2;
                c = c2;
                num = 3;
            } else {
                num = 2;
            }
            if (!push_frac(src2 * div, dst, false)) return false;
            double tb2 = (1.0 - src * div / dst) / tbw;
            if (tb2 > 45.0) tb2 = 45.0; // CDSPFIRFilter::getLPMaxTransBand()
            if (!push_bc(1.0 / num, tb2, num, num, 1)) return false;
            for (int k = 1; k < c; k++) push_hb(ST_HBUP, k - 1, num == 3);
        } else {
            if (!push_frac(src2, dst, false)) return false;
        }
        done = true;
    }

    if (!done) {
        // (4) downsampling with half-band decimators, :337-393
        double check = dst * 4.0;
        int c = 0;
        double fin_gain = 1.0;
        while (check <= src) {
            c++;
            check *= 2.0;
            fin_gain *= 0.5;
        }
        const int srdiv = (1 << c);
        int downf;
        double nf = 0.5;
        bool use_interp = true, third = false;
        for (downf = 2; downf <= 3 && !force_interp; downf++) {
            if (dst * srdiv * downf == src) {
                nf = 1.0 / downf;
                use_interp = false;
                third = (downf == 3);
                break;
            }
        }
        if (use_interp) {
            downf = 1;
            nf = dst * srdiv / src;
            third = (nf * 3.0 <= 1.0);
        }
        for (int k = 0; k < c; k++) push_hb(ST_HBDOWN, c - 1 - k, third);
        if (!push_bc(nf, tb, fin_gain, 1, downf)) return false;
        if (use_interp && !push_frac(src, dst * srdiv, third)) return false;
    }

    // Buffer-length chain (addProcessor, CDSPResampler.h:677-700).
    long long cur = max_in;
    for (size_t i = 0; i < stages.size(); i++) {
        cur = stage_max_out_len(stages[i], cur);
        if (!set_max_out_len(stages[i], i, cur, error)) return false;
    }
    max_out_len = (int) cur;
    return true;
}

bool Plan::build_trim(double src, double dst, int max_in, double tb, double att, int ext, double mt, bool any_pair)
{
    if (!(mt > 0.0 && mt <= 0.01)) {
        error = "max_trim must lie in (0, 0.01]";
        return false;
    }
    if (!build(src, dst, max_in, tb, att, 0, ext, 0, true, any_pair)) return false;
    if (passthrough) {
        error = "a passthrough rate pair (src == dst) has no interpolator whose ratio could be trimmed";
        passthrough = false;
        return false;
    }
    for (size_t i = 0; i < stages.size(); i++)
        if (stages[i].kind == ST_FRAC_POLY) trim_stage = (int) i;
    if (trim_stage < 0) {
        error = "this rate pair's chain has no fractional interpolator (an integer or power-of-two ratio); its ratio "
                "cannot be trimmed";
        return false;
    }
    max_trim = mt;
    // every buffer sized for the largest factor: the interpolator's bound at dsr(1 + max_trim), propagated down the chain
    long long cur = max_in;
    for (size_t i = 0; i < stages.size(); i++) {
        StageDesc& s = stages[i];
        if ((int) i == trim_stage) cur = (long long) std::ceil(cur * trim_dsr(1.0 + mt) / s.src_rate) + 1;
        else cur = stage_max_out_len(s, cur);
        if (!set_max_out_len(s, i, cur, error)) return false;
    }
    max_out_len = (int) cur;
    return true;
}

double Plan::trim_dsr(double f) const
{
    const StageDesc& s = stages[(size_t) trim_stage];
    return (dst_rate * f) * (s.dst_rate / dst_rate); // the second factor is 1 or the power of two srdiv, so exact
}

bool Plan::build_single(int kind, const double* a, int max_in, int ext)
{
    src_rate = 0;
    dst_rate = 0;
    max_in_len = max_in;
    extfft = ext ? 1 : 0;
    stages.clear();
    passthrough = false;
    error.clear();
    if (max_in > R8BGPU_MAX_LEN) {
        error = "MaxInLen " + std::to_string(max_in) + " is above R8BGPU_MAX_LEN = " + std::to_string(R8BGPU_MAX_LEN);
        return false;
    }
    StageDesc s;
    switch (kind) {
    case ST_BLOCKCONV:
        atten = a[2];
        trans_band = a[1];
        if (!make_blockconv(s, a[0], a[1], a[2], a[3], (int) a[4], (int) a[5], extfft, error)) return false;
        break;
    case ST_FRAC_WHOLE:
    case ST_FRAC_POLY:
        atten = a[2];
        if (!make_frac(s, a[0], a[1], a[2], a[3] != 0.0, 0, error)) return false;
        break;
    case ST_HBUP:
    case ST_HBDOWN:
        atten = a[0];
        make_hb(s, (StageKind) kind, a[0], (int) a[1], a[2] != 0.0);
        break;
    default:
        error = "unknown stage kind";
        return false;
    }
    if (!set_max_out_len(s, 0, stage_max_out_len(s, max_in), error)) return false;
    max_out_len = s.max_out_len;
    stages.push_back(std::move(s));
    return true;
}

int Plan::in_len_before_out_pos(int req_out_pos) const
{
    int req = req_out_pos;
    for (int c = (int) stages.size() - 1; c >= 0; c--)
        req = stage_in_len_before_out_pos(stages[(size_t) c], req);
    return req;
}

int Plan::input_required_for_output(int n) const
{
    if (n < 1) return 0;
    return in_len_before_out_pos(n - 1) + 1;
}

std::string Plan::describe() const
{
    char b[512];
    std::string r;
    snprintf(b, sizeof b, "* plan: src=%.1f dst=%.1f len=%i tb=%.1f att=%.2f extfft=%i\n", src_rate,
             dst_rate, max_in_len, trans_band, atten, extfft);
    r += b;
    for (const auto& s : stages) {
        switch (s.kind) {
        case ST_BLOCKCONV:
            snprintf(b, sizeof b, "BlockConv: flt_len=%i in_len=%i io=%i/%i latency=%i nfreq=%.4f gain=%.3f\n",
                     s.lp.kernel_len, s.ref_input_len, s.up, s.down, s.latency, s.norm_freq, s.gain);
            break;
        case ST_FRAC_WHOLE:
            snprintf(b, sizeof b, "FracInterp: src=%.2f dst=%.2f taps=%i whole step=%i/%i third=%i\n",
                     s.src_rate, s.dst_rate, s.bank.filter_len, s.in_step, s.out_step, (int) s.is_third);
            break;
        case ST_FRAC_POLY:
            snprintf(b, sizeof b, "FracInterp: src=%.2f dst=%.2f taps=%i fracs=%i order=2 third=%i\n",
                     s.src_rate, s.dst_rate, s.bank.filter_len, s.bank.fracs, (int) s.is_third);
            break;
        case ST_HBUP:
            snprintf(b, sizeof b, "HBUp: sti=%i third=%i taps=%i att=%.1f\n", s.steep_index,
                     (int) s.is_third, s.hb_taps, s.hb_atten);
            break;
        case ST_HBDOWN:
            snprintf(b, sizeof b, "HBDown: sti=%i third=%i taps=%i att=%.1f\n", s.steep_index,
                     (int) s.is_third, s.hb_taps, s.hb_atten);
            break;
        }
        r += b;
    }
    return r;
}

// ----------------------------------------------------------------------------------------------

void Schedule::init(const Plan* p)
{
    plan = p;
    poly.clear();
    clear();
}

void Schedule::clear()
{
    const size_t n = plan->stages.size();
    n_in.assign(n, 0);
    n_out.assign(n, 0);
    std::vector<PolyState> fresh(n); // InitFracPos == 0 for linear-phase chains (CDSPFracInterpolator.h:834-858)
    for (size_t i = 0; i < n; i++)
        fresh[i].dsr = i < poly.size() && poly[i].dsr != 0.0 ? poly[i].dsr : plan->stages[i].dst_rate;
    poly.swap(fresh);
}

bool Schedule::retime(double dsr)
{
    PolyState& ps = poly[(size_t) plan->trim_stage];
    if (memcmp(&ps.dsr, &dsr, sizeof dsr) == 0) return false;
    ps.dsr = dsr;
    ps.in_counter = 0;
    ps.in_pos_int = 0;
    ps.in_pos_shift = ps.fpos * dsr / plan->stages[(size_t) plan->trim_stage].src_rate;
    return true;
}

namespace {

// Position of the k-th output after the call-start state (k >= 1); mirrors the reference's
// expression order exactly: ((InCounter + InPosShift) * ssr) / dsr   (CDSPFracInterpolator.h:1161-1166)
inline void poly_pos(const Schedule::PolyState& st, double ssr, double dsr, long long k,
                     long long& p, int& ni, double& fpos)
{
    const int ic = st.in_counter + (int) k;
    const double next_pos = (ic + st.in_pos_shift) * ssr / dsr;
    ni = (int) next_pos;
    p = st.p + (ni - st.in_pos_int);
    fpos = next_pos - ni;
}

} // namespace

int Schedule::advance(int l, std::vector<StageCall>& calls)
{
    const auto& st = plan->stages;
    calls.assign(st.size(), StageCall());
    long long feed0 = 0, feed1 = 0;
    for (size_t i = 0; i < st.size(); i++) {
        StageCall& c = calls[i];
        if (i == 0) {
            c.n0 = n_in[0];
            c.n1 = n_in[0] + l;
        } else {
            c.n0 = feed0;
            c.n1 = feed1;
        }
        c.e0 = n_out[i];
        const StageDesc& s = st[i];
        long long e1 = c.e0;
        switch (s.kind) {
        case ST_BLOCKCONV: e1 = blockconv_emitted(s, c.n1); break;
        case ST_FRAC_WHOLE: e1 = frac_whole_emitted(s, c.n1); break;
        case ST_HBUP: e1 = hbup_emitted(s, c.n1); break;
        case ST_HBDOWN: e1 = hbdown_emitted(s, c.n1); break;
        case ST_FRAC_POLY: {
            PolyState& ps = poly[i];
            const double ssr = s.src_rate, dsr = ps.dsr;
            c.in_counter0 = ps.in_counter;
            c.in_pos_int0 = ps.in_pos_int;
            c.in_pos_shift = ps.in_pos_shift;
            c.fpos0 = ps.fpos;
            c.p0 = ps.p;
            c.ssr = ssr;
            c.dsr = dsr;
            const long long fl2 = s.bank.filter_len / 2;
            const long long pmax = c.n1 - 1 - fl2; // produce while p <= pmax
            long long cnt = 0;
            if (s.fasttiming) {
                // CDSPFracInterpolator.h:1153-1158: fpos += FracStep; PosIncr = (int) fpos; fpos -= PosIncr
                const double frac_step = s.src_rate / s.dst_rate; // :713
                c.p_last = ps.p;
                while (ps.p <= pmax) {
                    c.ft_dp.push_back((int) (ps.p - c.p0));
                    c.ft_fpos.push_back(ps.fpos);
                    c.p_last = ps.p;
                    cnt++;
                    ps.fpos += frac_step;
                    const int inc = (int) ps.fpos;
                    ps.fpos -= inc;
                    ps.p += inc;
                }
                e1 = c.e0 + cnt;
                break;
            }
            if (ps.p <= pmax) {
                // largest k with p_k <= pmax (p_k is non-decreasing in k); k = 0 qualifies.
                long long lo = 0;
                long long hi = (long long) ((double) (pmax - ps.p + 2) * dsr / ssr) + 4;
                auto pk = [&](long long k) {
                    long long p;
                    int ni;
                    double f;
                    poly_pos(ps, ssr, dsr, k, p, ni, f);
                    return p;
                };
                while (pk(hi) <= pmax) hi *= 2;
                while (hi - lo > 1) {
                    const long long mid = lo + (hi - lo) / 2;
                    if (pk(mid) <= pmax) lo = mid;
                    else hi = mid;
                }
                cnt = lo + 1;
            }
            e1 = c.e0 + cnt;
            c.p_last = ps.p;
            if (cnt > 1) {
                long long p;
                int ni;
                double f;
                poly_pos(ps, ssr, dsr, cnt - 1, p, ni, f);
                c.p_last = p;
            }
            if (cnt > 0) {
                long long p;
                int ni;
                double f;
                poly_pos(ps, ssr, dsr, cnt, p, ni, f);
                ps.in_counter += (int) cnt;
                ps.p = p;
                ps.in_pos_int = ni;
                ps.fpos = f;
            }
            if (ps.in_counter > 1000) { // once per process() call, CDSPFracInterpolator.h:907-919
                ps.in_counter = 0;
                ps.in_pos_int = 0;
                ps.in_pos_shift = ps.fpos * dsr / ssr;
            }
            break;
        }
        }
        c.e1 = e1;
        n_in[i] = c.n1;
        n_out[i] = e1;
        feed0 = c.e0;
        feed1 = c.e1;
    }
    if (st.empty()) return l;
    return (int) (calls.back().e1 - calls.back().e0);
}

// ----------------------------------------------------------------------------------------------

namespace {

// the whole state of a schedule as one ordered key (doubles by bit pattern: equal keys advance bit-identically)
std::vector<long long> state_key(const Schedule& s)
{
    std::vector<long long> k;
    k.reserve(s.n_in.size() * 8);
    k.insert(k.end(), s.n_in.begin(), s.n_in.end());
    k.insert(k.end(), s.n_out.begin(), s.n_out.end());
    for (const Schedule::PolyState& p : s.poly) {
        long long a, b, d;
        memcpy(&a, &p.in_pos_shift, sizeof a);
        memcpy(&b, &p.fpos, sizeof b);
        memcpy(&d, &p.dsr, sizeof d);
        k.push_back(p.in_counter);
        k.push_back(p.in_pos_int);
        k.push_back(a);
        k.push_back(b);
        k.push_back(p.p);
        k.push_back(d);
    }
    return k;
}

} // namespace

bool same_state(const Schedule& a, const Schedule& b) { return state_key(a) == state_key(b); }

void RaggedSchedule::init(const Schedule& lockstep, int n_ch)
{
    groups.assign(1, lockstep);
    group_of.assign((size_t) n_ch, 0);
}

void RaggedSchedule::plan_call(const int* lens, Step& step) const
{
    const int n_ch = (int) group_of.size();
    step = Step();
    step.key_of.resize((size_t) n_ch);
    std::map<std::pair<int, int>, int> keys;
    for (int c = 0; c < n_ch; c++) {
        const std::pair<int, int> gk(group_of[(size_t) c], lens[c]);
        auto it = keys.find(gk);
        if (it == keys.end()) {
            const int k = (int) step.next.size();
            it = keys.emplace(gk, k).first;
            step.next.push_back(groups[(size_t) gk.first]);
            step.calls.emplace_back();
            step.len.push_back(lens[c]);
            step.count.push_back(step.next.back().advance(lens[c], step.calls.back()));
        }
        step.key_of[(size_t) c] = it->second;
        if (!step.runs.empty() && step.runs.back().key == it->second) step.runs.back().n++;
        else step.runs.push_back(Run{c, 1, it->second});
    }
}

void RaggedSchedule::merge(std::vector<Schedule>& g, std::vector<int>& of)
{
    std::map<std::vector<long long>, int> seen;
    std::vector<int> remap(g.size());
    std::vector<Schedule> out;
    for (size_t i = 0; i < g.size(); i++) {
        auto r = seen.emplace(state_key(g[i]), (int) out.size());
        if (r.second) out.push_back(g[i]);
        remap[i] = r.first->second;
    }
    for (int& x : of) x = remap[(size_t) x];
    // drop groups no channel is in
    std::vector<int> used(out.size(), -1);
    std::vector<Schedule> live;
    for (int& x : of) {
        if (used[(size_t) x] < 0) {
            used[(size_t) x] = (int) live.size();
            live.push_back(out[(size_t) x]);
        }
        x = used[(size_t) x];
    }
    g.swap(live);
}

void RaggedSchedule::commit(const Step& step)
{
    groups = step.next;
    group_of = step.key_of;
    merge(groups, group_of);
}

void RaggedSchedule::clear_channels(const int* ch, int n)
{
    if (n <= 0 || groups.empty()) return;
    // one fresh schedule per group a named channel leaves: each keeps its interpolator's dsr (a trim factor)
    std::map<int, int> fresh;
    for (int i = 0; i < n; i++) {
        int& g = group_of[(size_t) ch[i]];
        auto it = fresh.find(g);
        if (it == fresh.end()) {
            it = fresh.emplace(g, (int) groups.size()).first;
            groups.push_back(groups[(size_t) g]);
            groups.back().clear();
        }
        g = it->second;
    }
    merge(groups, group_of);
}

void RaggedSchedule::retime_channels(const int* ch, int n, const double* dsr)
{
    if (n <= 0 || groups.empty()) return;
    std::map<std::pair<int, unsigned long long>, int> moved; // (group, dsr bits) -> its retimed copy
    for (int i = 0; i < n; i++) {
        int& g = group_of[(size_t) ch[i]];
        unsigned long long bits;
        memcpy(&bits, &dsr[i], sizeof bits);
        const std::pair<int, unsigned long long> key(g, bits);
        auto it = moved.find(key);
        if (it == moved.end()) {
            Schedule s = groups[(size_t) g];
            if (!s.retime(dsr[i])) continue; // the same factor again: no re-base
            it = moved.emplace(key, (int) groups.size()).first;
            groups.push_back(s);
        }
        g = it->second;
    }
    merge(groups, group_of);
}

void RaggedSchedule::install(const int* ch, int n, const Schedule* s)
{
    if (n <= 0 || groups.empty()) return;
    for (int i = 0; i < n; i++) {
        group_of[(size_t) ch[i]] = (int) groups.size();
        groups.push_back(s[i]);
    }
    merge(groups, group_of); // equal schedules share a group again, whatever slot or batch they came from
}

// ----------------------------------------------------------------------------------------------

void plan_flush(const Schedule& s, long long target, FlushPlan& f, bool keep_calls)
{
    f = FlushPlan();
    f.target = target;
    if (target <= s.outputs()) return;
    f.count = (int) (target - s.outputs());
    const int M = s.plan->max_in_len;
    Schedule w = s, t = s; // assignments between equal-sized schedules reuse their storage
    std::vector<StageCall> calls;
    while (true) {
        t = w;
        t.advance(M, calls);
        if (t.outputs() < target) { // a whole sub-step of silence does not reach the target
            if (keep_calls) {
                f.lens.push_back(M);
                f.calls.push_back(calls);
            }
            f.zeros += M;
            std::swap(w, t);
            continue;
        }
        // the shortest last sub-step that does (the chain's output count never decreases with its input length):
        // outputs after lo samples < target <= outputs after hi samples
        int lo = 0, hi = M;
        while (hi - lo > 1) {
            const int mid = lo + (hi - lo) / 2;
            t = w;
            t.advance(mid, calls);
            (t.outputs() < target ? lo : hi) = mid;
        }
        t = w;
        t.advance(hi, calls);
        // The last stage stops at the target (the stream is cleared afterwards).  A half-band upsampler writes its
        // outputs in pairs (2n, 2n + 1) from an even e0, so its range must stay even: it stops at the target rounded up
        // to even, and the caller keeps the spare sample out of the caller's buffer (r8b_capi.cu, run_flush).
        StageCall& last = calls.back();
        last.e1 = s.plan->stages.back().kind == ST_HBUP ? std::min(last.e1, target + (target & 1)) : target;
        if (keep_calls) {
            f.lens.push_back(hi);
            f.calls.push_back(calls);
        }
        f.zeros += hi;
        return;
    }
}

namespace {

int bit_len(unsigned __int128 v)
{
    int n = 0;
    while (v != 0) {
        v >>= 1;
        n++;
    }
    return n;
}

} // namespace

long long flush_default_target(const Plan& p, long long n_in)
{
    if (n_in <= 0) return 0;
    // each rate is m * 2^e with an integer m < 2^53: dst / src = (b / a) * 2^sh exactly
    int es = 0, ed = 0;
    unsigned long long a = (unsigned long long) std::ldexp(std::frexp(p.src_rate, &es), 53);
    unsigned long long b = (unsigned long long) std::ldexp(std::frexp(p.dst_rate, &ed), 53);
    int sh = ed - es;
    while ((a & 1) == 0) {
        a >>= 1;
        sh--;
    }
    while ((b & 1) == 0) {
        b >>= 1;
        sh++;
    }
    unsigned __int128 num = (unsigned __int128) n_in * b, den = a; // num < 2^116
    if (sh >= 0) {
        if (bit_len(num) + sh > 126) return -1;
        num <<= sh;
    } else {
        if (bit_len(den) - sh > 126) return 1; // den > 2^126 > num > 0
        den <<= -sh;
    }
    const unsigned __int128 q = (num + den - 1) / den;
    return q > (unsigned __int128) LLONG_MAX ? -1 : (long long) q;
}

// Every stage's emitted count is bounded below by a line in its input count n (r8b_plan.h formulas):
//   BlockConv   ceil((U n - Latency) / D)        >= (U/D) n - Latency/D
//   FracWhole   (n - fl2) OutStep/InStep rounded  >= (OutStep/InStep) n - fl2 OutStep/InStep
//   FracPoly    #{k : pos_k <= n - 1 - fl2}       >= (dst/src) n - (fl2 + 2) dst/src - 1   (pos_k = floor(k src/dst) up
//                                                   to the rounding of the timing arithmetic, far below one sample)
//   HBUp        2 (n - T)                         >= 2 n - 2 T
//   HBDown      floor(n / 2) - (T - 1)            >= n / 2 - (T - 1/2)
// Emission never decreases with the input, so the lines compose: after N inputs the chain has produced at least
// R N - C samples, R = dst/src (the product of the stage ratios), C = sum over stages of c_i times the ratios after it.
// A default flush returns ceil(N R) - outputs <= C + 1; one more sample covers the rounding of C.
int flush_max_out_len(const Plan& p)
{
    if (p.passthrough) return 0;
    double c = 0.0;
    for (const StageDesc& s : p.stages) {
        double r = 1.0, ci = 0.0;
        switch (s.kind) {
        case ST_BLOCKCONV:
            r = (double) s.up / s.down;
            ci = (double) s.latency / s.down;
            break;
        case ST_FRAC_WHOLE:
            r = (double) s.out_step / s.in_step;
            ci = (s.bank.filter_len / 2) * r;
            break;
        case ST_FRAC_POLY:
            r = s.dst_rate / s.src_rate;
            ci = (s.bank.filter_len / 2 + 2) * r + 1.0;
            break;
        case ST_HBUP:
            r = 2.0;
            ci = 2.0 * s.hb_taps;
            break;
        case ST_HBDOWN:
            r = 0.5;
            ci = s.hb_taps - 0.5;
            break;
        }
        c = c * r + ci;
    }
    return (int) std::ceil(c) + 2;
}

} // namespace r8bgpu

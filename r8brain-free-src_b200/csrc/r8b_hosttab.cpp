// r8b_hosttab.cpp -- see r8b_hosttab.h.
#include "r8b_hosttab.h"

#include "r8b_fused2_core.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "r8b_bclarge.cuh"
#include "r8b_fft.cuh"

namespace r8bgpu {

namespace {
// Spectrum of the polyphase-packed filter in FFT slot order (see k_blockconv).
template <int M>
void fill_slot_order(const std::vector<double2>& nat, std::vector<double2>& out)
{
    out.resize((size_t) M);
    for (int k = 0; k < M; k++) out[(size_t) slot_of<M>(k)] = nat[(size_t) k];
}

} // namespace

void build_spectrum(const StageDesc& s, int fft_log2, std::vector<double2>& spec_slots,
                    std::vector<double2>& tw, double* nyq_gain)
{
    const int M = 1 << fft_log2;
    const int L = s.lp.half_len, U = (s.up > 2) ? 1 : s.up; // up = 3 runs on the zero-stuffed stream
    const long double two_pi = 6.283185307179586476925286766559005768L;
    std::vector<long double> cs((size_t) M), sn((size_t) M);
    for (int k = 0; k < M; k++) {
        // exact octant symmetries are not needed at long-double accuracy
        const long double a = two_pi * (long double) k / (long double) M;
        cs[(size_t) k] = cosl(a);
        sn[(size_t) k] = sinl(a);
    }
    tw.resize((size_t) M);
    for (int k = 0; k < M; k++) tw[(size_t) k] = make_double2((double) cs[(size_t) k], (double) -sn[(size_t) k]);

    // g[j] = h[U*j] + i*h[U*j+1] (U==2) or h[j] (U==1), j in [-lg, lg]
    const int lg = (L + U - 1) / U;
    const double* h = s.lp.taps.data() + L; // h[-L..L]
    auto tap = [&](long long idx) -> long double {
        return (idx < -L || idx > L) ? 0.0L : (long double) h[idx];
    };
    const long double scale = 1.0L / ((long double) M * (U == 2 ? 2.0L : 1.0L));
    std::vector<double2> nat((size_t) M);
    for (int k = 0; k < M; k++) {
        long double re = 0.0L, im = 0.0L;
        for (int j = -lg; j <= lg; j++) {
            const long double gr = tap((long long) U * j);
            const long double gi = (U == 2) ? tap((long long) U * j + 1) : 0.0L;
            if (gr == 0.0L && gi == 0.0L) continue;
            const int idx = (int) ((((long long) j * k) % M + M) % M);
            const long double c = cs[(size_t) idx], sv = -sn[(size_t) idx]; // exp(-i*2pi*j*k/M)
            re += gr * c - gi * sv;
            im += gr * sv + gi * c;
        }
        nat[(size_t) k] = make_double2((double) (re * scale), (double) (im * scale));
    }
    if (s.block_exact) {
        // Power-of-two decimation in the reference = inverse transform of only the lowest 1/D of
        // the block spectrum (CDSPBlockConvolver.h:329-344).  Same thing here: the bins that the
        // shorter inverse FFT never sees are zeroed and the full-length inverse is sampled every
        // D-th point.  (The folded Nyquist term kb[z]*p[z]-kb[z+1]*p[z+1] is the product of two
        // stop-band values, far below one ulp of the output, and is dropped.)
        const int keep = M / (2 * s.down);
        if (nyq_gain) *nyq_gain = nat[(size_t) keep].x;
        for (int k = keep; k <= M - keep; k++) nat[(size_t) k] = make_double2(0.0, 0.0);
    }
    switch (fft_log2) {
    case 6: fill_slot_order<64>(nat, spec_slots); break;
    case 7: fill_slot_order<128>(nat, spec_slots); break;
    case 8: fill_slot_order<256>(nat, spec_slots); break;
    case 9: fill_slot_order<512>(nat, spec_slots); break;
    case 10: fill_slot_order<1024>(nat, spec_slots); break;
    case 11: fill_slot_order<2048>(nat, spec_slots); break;
    case 13: fill_slot_order<8192>(nat, spec_slots); break;
    default: fill_slot_order<4096>(nat, spec_slots); break;
    }
}

void build_spectrum_large(const StageDesc& s, int fft_log2, std::vector<double2>& spec_slots, std::vector<double2>& tw4096,
                          std::vector<double2>& tw_m, double* nyq_gain)
{
    const int M = 1 << fft_log2, R0 = M / bcl::SUB, L = s.lp.half_len;
    const long double two_pi = 6.283185307179586476925286766559005768L;
    std::vector<long double> cs((size_t) M), sn((size_t) M);
    for (int k = 0; k < M; k++) {
        const long double a = two_pi * (long double) k / (long double) M;
        cs[(size_t) k] = cosl(a);
        sn[(size_t) k] = sinl(a);
    }
    tw_m.resize((size_t) M);
    for (int k = 0; k < M; k++) tw_m[(size_t) k] = make_double2((double) cs[(size_t) k], (double) -sn[(size_t) k]);
    tw4096.resize((size_t) bcl::SUB);
    for (int k = 0; k < bcl::SUB; k++) tw4096[(size_t) k] = tw_m[(size_t) k * R0];

    // H[k] = h[0] + sum_j (h[j] + h[-j]) cos(2 pi jk/M) - i (h[j] - h[-j]) sin(2 pi jk/M), j = 1..L (the designed kernel
    // is symmetric, so the sine sum is skipped when every difference is zero)
    const double* h = s.lp.taps.data() + L; // h[-L..L]
    std::vector<long double> hs((size_t) L + 1), hd((size_t) L + 1);
    bool odd_part = false;
    for (int j = 1; j <= L; j++) {
        hs[(size_t) j] = (long double) h[j] + (long double) h[-j];
        hd[(size_t) j] = (long double) h[j] - (long double) h[-j];
        odd_part = odd_part || hd[(size_t) j] != 0.0L;
    }
    const long double scale = 1.0L / (long double) M;
    // reference-exact decimation keeps bins [0, M/(2D)) and (M - M/(2D), M) plus the Nyquist gain at M/(2D)
    const int keep = s.block_exact ? M / (2 * s.down) : M / 2;
    std::vector<double2> nat((size_t) M, make_double2(0.0, 0.0));
    for (int k = 0; k <= keep; k++) {
        long double re = (long double) h[0], im = 0.0L;
        unsigned idx = 0;
        for (int j = 1; j <= L; j++) {
            idx = (idx + (unsigned) k) & (unsigned) (M - 1); // j k mod M
            re += hs[(size_t) j] * cs[idx];
            if (odd_part) im -= hd[(size_t) j] * sn[idx];
        }
        nat[(size_t) k] = make_double2((double) (re * scale), (double) (im * scale));
    }
    for (int k = 1; k < keep; k++) nat[(size_t) (M - k)] = make_double2(nat[(size_t) k].x, -nat[(size_t) k].y);
    if (s.block_exact) {
        if (nyq_gain) *nyq_gain = nat[(size_t) keep].x;
        nat[(size_t) keep] = make_double2(0.0, 0.0);
    }
    spec_slots.resize((size_t) M);
    for (int k = 0; k < M; k++) spec_slots[(size_t) bcl::slot_of_large(k, R0)] = nat[(size_t) k];
}

int choose_fft_log2(int lg, int min_log2, int max_log2)
{
    if (const char* e = getenv("R8BGPU_FFT_LOG2")) {
        const int v = atoi(e);
        if (v >= min_log2 && v <= max_log2 && (1 << v) - 2 * lg >= 64) return v;
    }
    int best = -1;
    double best_cost = 0.0;
    for (int b = min_log2; b <= max_log2; b++) {
        const int m = 1 << b;
        const int valid = m - 2 * lg;
        if (valid < 64) continue;
        const double cost = (double) b * m / valid;
        if (best < 0 || cost < best_cost) {
            best = b;
            best_cost = cost;
        }
    }
    return best;
}

void blockconv_call_fields(BlockConvParams& p, const StageDesc& s, int virt_up, int lg, int fft_log2, long long e0, long long e1)
{
    const int up_eff = virt_up > 1 ? 1 : s.up;
    p.up = up_eff;
    p.src_up = virt_up;
    p.down = s.down;
    p.lg = lg;
    p.fft_log2 = fft_log2;
    p.e0 = e0;
    p.e1 = e1;
    p.m0 = (e0 * s.down) / up_eff;             // floor; indices are >= 0
    p.m1 = ((e1 - 1) * s.down) / up_eff + 1;
    if (s.block_exact) {
        // tile b = reference block b: owns positions [b*InputLen - L, (b+1)*InputLen - L)
        const long long il = s.ref_input_len, L = s.lp.half_len;
        const long long b0 = (p.m0 + L) / il, b1 = (p.m1 - 1 + L) / il;
        p.m0 = b0 * il - L;
        p.adv = (int) il;
        p.n_tiles = (int) (b1 - b0 + 1);
    } else {
        const int adv_max = (1 << fft_log2) - 2 * lg;
        const long long span = p.m1 - p.m0;
        long long nt = (span + adv_max - 1) / adv_max;
        if (nt > 1 && (nt & 1)) nt++; // tiles are transformed in pairs
        p.n_tiles = (int) nt;
        p.adv = (int) ((span + nt - 1) / nt);
    }
    p.trunc = s.block_exact ? s.down : 0;
    p.nyq_gain = 0.0;
    p.spec = nullptr;
    p.tw = nullptr;
}

BcTile blockconv_tile(const StageDesc& s, bool allow_large)
{
    BcTile t;
    // up-factors other than 1 and 2 (the planner only makes 3) run as a 1x convolution over the zero-stuffed stream,
    // exactly as the reference does
    t.virt_up = (s.up > 2) ? s.up : 1;
    t.up = (s.up > 2) ? 1 : s.up;
    t.lg = (s.lp.half_len + t.up - 1) / t.up;
    t.fft_log2 = choose_fft_log2(t.lg, 10, t.up == 1 ? 13 : 12);
    if (s.block_exact) { // tiles == the reference's own blocks (2 << BlockLenBits)
        t.lg = s.ref_prev_len - s.lp.half_len;
        t.fft_log2 = s.lp.block_len_bits + 1;
        const int lo = t.up == 1 ? 6 : 10, hi = t.up == 1 ? 13 : 12;
        if (t.fft_log2 >= lo && t.fft_log2 <= hi) return t;
        t.large = allow_large && t.up == 1 && t.fft_log2 >= 14 && t.fft_log2 <= 16;
        if (!t.large) t.fft_log2 = -1;
        return t;
    }
    if (t.fft_log2 >= 0 || !allow_large) return t;
    // too long for the in-shared-memory tiles: a 1x convolution over the (zero-stuffed) stream on large tiles
    if (t.up == 2) {
        t.virt_up = 2;
        t.up = 1;
        t.lg = s.lp.half_len;
    }
    t.fft_log2 = choose_fft_log2(t.lg, 14, 16);
    t.large = t.fft_log2 >= 0;
    return t;
}


std::vector<double2> build_tw_tab(const std::vector<double2>& tw)
{
    std::vector<double2> tt(512);
    for (int q = 0; q < 16; q++)
        for (int r = 0; r < 16; r++) {
            tt[(size_t) (q * 16 + r)] = tw[(size_t) ((r * q) * 16)];   // W_256^(r q) = W_4096^(16 r q)
            tt[(size_t) (256 + q * 16 + r)] = tw[(size_t) (r * q)];    // W_4096^(r q)
        }
    return tt;
}

std::vector<double2> build_c_tab(const std::vector<double2>& spec, const std::vector<double2>& tw, int up)
{
    using namespace f2;
    if (up == 1) {
        // H[k]/2 for k = 0..N from the slot-ordered table of FFT(h)/M (the halving is exact)
        auto hk = [&](int k) {
            const double2 v = spec[(size_t) slot_of<FM>(k)];
            return make_double2(0.5 * v.x, 0.5 * v.y);
        };
        std::vector<double2> ct((size_t) 4 * 3 * HT + 3);
        for (int u = 0; u < 4; u++)
            for (int ht = 0; ht < HT; ht++) {
                const int k = c_freq(ht, u);
                double2* e = &ct[(size_t) (u * 3) * HT + ht];
                e[0] = tw[(size_t) k];
                e[HT] = hk(k);
                e[2 * HT] = hk(FN - k); // k = 0: the Nyquist bin
            }
        ct[(size_t) 12 * HT] = tw[(size_t) (FN / 2)];
        ct[(size_t) 12 * HT + 1] = hk(FN / 2);
        ct[(size_t) 12 * HT + 2] = hk(FN / 2);
        return ct;
    }
    return std::vector<double2>(); // up 2: phase C runs inside the first inverse pass (build_cd_tab)
}

std::vector<double2> build_cd_tab(const std::vector<double2>& spec, const std::vector<double2>& tw)
{
    using namespace f2;
    std::vector<double2> ct((size_t) 17 * HT);
    for (int g = 0; g < HT; g++) {
        for (int q3 = 0; q3 < 16; q3++) ct[(size_t) q3 * HT + g] = spec[(size_t) (16 * g + q3)];
        ct[(size_t) 16 * HT + g] = tw[(size_t) ((g >> 4) + 16 * (g & 15))];
    }
    return ct;
}

std::vector<double2> build_cs_tab(const StageDesc& s, const std::vector<double2>& tw)
{
    using namespace f2;
    // a0[k] = sum_j h[2j] cos(2 pi j k / M) / (2M),  a1[k] = sum_j h[2j+1] cos(pi (2j+1) k / M) / (2M), k = 0..N, each
    // summed in long double over every tap of the (zero-phase) kernel and rounded once
    constexpr int M = FM, M2 = 2 * FM;
    const int L = s.lp.half_len;
    const double* h = s.lp.taps.data() + L; // h[-L..L]
    const long double pi = 3.141592653589793238462643383279502884L;
    std::vector<long double> cs((size_t) M2);
    for (int m = 0; m < M2; m++) cs[(size_t) m] = cosl(pi * (long double) m / (long double) M); // cos(2 pi m / 2M)
    const long double scale = 1.0L / (2.0L * (long double) M);
    std::vector<double2> ct((size_t) CS_PAIRS + 2 * HT);
    for (int k = 0; k <= FN; k++) {
        long double a0 = 0.0L, a1 = 0.0L;
        for (int n = -L; n <= L; n++) { // tap n = 2j (g0) or 2j + 1 (g1): the angle is pi n k / M either way
            const long double v = (long double) h[n] * cs[(size_t) ((((long long) n * k) % M2 + M2) % M2)];
            if (n & 1) a1 += v;
            else a0 += v;
        }
        ct[(size_t) cs_entry(k)] = make_double2((double) (a0 * scale), (double) (a1 * scale));
    }
    for (int g = 0; g < HT; g++) {
        const int k0 = (g >> 4) + 16 * (g & 15);
        ct[(size_t) CS_PAIRS + g] = tw[(size_t) k0];
        ct[(size_t) CS_PAIRS + HT + g] = make_double2((double) cs[(size_t) k0], (double) sinl(pi * (long double) k0 / (long double) M));
    }
    return ct;
}

int fused2_smem_bytes(int bank_doubles, bool cs, bool staged)
{
    using namespace f2;
    return 2 * FPL2 * (int) sizeof(double2) + 512 * (int) sizeof(double2) + ((bank_doubles + 1) & ~1) * (int) sizeof(double) +
           (cs ? CS_PAIRS * (int) sizeof(double2) : 0) + (staged ? (2 * HT / 32) * 256 * (int) sizeof(double) : 0);
}

int fused2_stage_off(int bank_doubles, bool cs) { return fused2_smem_bytes(bank_doubles, cs, false) / (int) sizeof(double); }

int fused2_bank_doubles_max(const StageDesc& f)
{
    if (f.kind != ST_FRAC_WHOLE) return 0;
    const GroupBank tc = build_group_bank(f, 8, true), fma = build_group_bank(f, choose_group_ir(f), false);
    return std::max(tc.n_groups * tc.smaxp * tc.ir, fma.n_groups * fma.smaxp * fma.ir);
}

bool fused2_cs_fits(int bank_doubles_max) { return fused2_smem_bytes(bank_doubles_max, true, false) <= kFused2SmemMax; }

std::vector<double2> build_c_tab_v1(const std::vector<double2>& spec)
{
    constexpr int NT = 512, NC = FM / (2 * NT);
    std::vector<double2> ct((size_t) NC * 2 * NT);
    for (int u = 0; u < NC; u++)
        for (int tid = 0; tid < NT; tid++) {
            const int s1 = 16 * ((tid >> 3) + 64 * u) + (tid & 7);
            const int k = freq_of<FM>(s1);
            const int s2 = slot_of<FM>((FM - k) & (FM - 1));
            ct[(size_t) (2 * u) * NT + tid] = spec[(size_t) s1];
            ct[(size_t) (2 * u + 1) * NT + tid] = spec[(size_t) s2];
        }
    return ct;
}

FusedGeom fused_geometry(const StageDesc& s, const StageDesc& f)
{
    FusedGeom g;
    if (!(s.kind == ST_BLOCKCONV && (s.up == 2 || s.up == 1) && s.down == 1 && !s.block_exact &&
          (f.kind == ST_FRAC_WHOLE || (f.kind == ST_FRAC_POLY && s.up == 2))))
        return g;
    g.up = s.up;
    // half support of the filter as seen from one tile sample: polyphase branches for up 2 (input-rate samples)
    const int lg = s.up == 2 ? (s.lp.half_len + 1) / 2 : s.lp.half_len;
    const int flen = f.bank.filter_len, fll = flen / 2 - 1;
    int dmax = 0;
    if (f.kind == ST_FRAC_WHOLE)
        dmax = (int) (((long long) 9 * f.in_step + f.out_step - 1) / f.out_step) + 1; // up to 10 phases per group
    const int yl = (fll + 2) & ~1;
    const int yr = (dmax + flen - yl + 2 + 1) & ~1;
    // stream positions a tile can own: the valid part of its (up * 4096)-sample window minus the interpolation margins
    const int smax = (s.up * (4096 - 2 * lg) - yl - yr) & ~1;
    if (!(smax >= 1024 && (f.kind == ST_FRAC_POLY || f.in_step < smax / 2))) return g;
    g.ok = true;
    g.lg = lg;
    g.yl = yl;
    g.yr = yr;
    g.span_max = smax;
    g.ysh = 31;
    if (f.kind == ST_FRAC_WHOLE && (f.in_step & 1) == 0) {
        // lanes step by in_step doubles through the tile: make the padded stride odd
        int sh = 0;
        while (((f.in_step >> sh) & 1) == 0) sh++;
        g.ysh = sh < 4 ? 4 : sh;
        if (((f.in_step + (f.in_step >> g.ysh)) & 1) == 0) g.ysh = 31; // cannot fix; accept conflicts
    }
    return g;
}

// IR is 8 or 10, whichever spreads the phase groups more evenly over 16 warps (v1) / pairs of groups over 8 (v2).
int choose_group_ir(const StageDesc& s)
{
    int ir = 8;
    const int g8 = (s.out_step + 7) / 8, g10 = (s.out_step + 9) / 10;
    const int c8 = ((g8 + 15) / 16) * 8, c10 = ((g10 + 15) / 16) * 10;
    // measured (v1): the 10-phase variant spills registers; where 8-phase groups can start every call on a 64-byte
    // output boundary (out_step % 8 == 0: cfg 2) it loses by ~4 % despite the even task split, elsewhere the split
    // wins (cfg 3, out_step 147: 1.88 vs 1.98 ms)
    if (s.out_step % 8 != 0 && c10 < c8) ir = 10;
    if (const char* e = getenv("R8BGPU_IR")) ir = atoi(e) == 10 ? 10 : 8;
    return ir;
}

GroupBank build_group_bank(const StageDesc& s, int ir, bool frag_order)
{
    GroupBank B;
    const int os = s.out_step, flen = s.bank.filter_len;
    B.ir = ir;
    B.off.resize((size_t) os);
    B.row.resize((size_t) os);
    for (int r = 0; r < os; r++) {
        const long long pos = (long long) r * s.in_step;
        B.off[(size_t) r] = (int) (pos / os);
        B.row[(size_t) r] = (int) (pos % os);
    }
    B.n_groups = (os + ir - 1) / ir;
    // window offset of "phase" pr >= 0 counted from cycle 0 (pr >= os continues in later cycles)
    auto offx = [&](int pr) { return B.off[(size_t) (pr % os)] + (pr / os) * s.in_step; };
    int dmax = 0;
    for (int r0 = 0; r0 < os; r0++) dmax = std::max(dmax, offx(r0 + ir - 1) - offx(r0));
    B.smaxp = (flen + dmax + 3) & ~3;
    // one entry per possible first phase r0: lets a call start its groups at e0 mod 8
    B.gb.assign((size_t) os * B.smaxp * ir, 0.0);
    B.go.resize((size_t) os);
    for (int r0 = 0; r0 < os; r0++) {
        B.go[(size_t) r0] = B.off[(size_t) r0];
        for (int r = 0; r < ir; r++) {
            const int pr = r0 + r;
            const int dr = offx(pr) - offx(r0);
            const double* rowp = s.bank.table.data() + (size_t) B.row[(size_t) (pr % os)] * flen;
            for (int i = 0; i < flen; i++) {
                const int tap = dr + i;
                const size_t at = frag_order ? (size_t) (tap & ~3) * 8 + (size_t) r * 4 + (tap & 3) : (size_t) tap * ir + r;
                B.gb[(size_t) r0 * B.smaxp * ir + at] = rowp[i];
            }
        }
    }
    return B;
}

void fused_whole_fields(FusedParams& p, const StageDesc& f, long long e0, long long e1)
{
    p.mode = 0;
    p.flen = f.bank.filter_len;
    p.fll = p.flen / 2 - 1;
    p.e0 = e0;
    p.e1 = e1;
    p.in_step = f.in_step;
    p.out_step = f.out_step;
    p.p_lo = ((e0 * f.in_step) / f.out_step) & ~1LL; // even (positions are >= 0)
    p.p_hi = ((e1 - 1) * f.in_step) / f.out_step + 1;
    // groups of 8 phases start at e0 mod 8: every 64-byte output row is then aligned in the caller's buffer
    p.wrap = (f.out_step % 8 == 0 && !getenv("R8BGPU_NO_ALIGN")) ? 1 : 0;
    p.delta = p.wrap ? (int) (e0 & 7) : 0;
}

void fused2_tiles(FusedParams& p, const FusedGeom& g, int cur_parity)
{
    // One tile per half-CTA, no pairing.  Spans are multiples of 4 so that every tile's FFT window starts on the
    // same parity of the input index, and p_lo gives way by one sample pair where that makes the windows start
    // 16-byte aligned in the caller's block.
    const long long w0 = (g.up == 1 ? p.p_lo - g.yl : (p.p_lo - g.yl) / 2) - g.lg;
    const int back = g.up == 1 ? 1 : 2; // stream positions per input sample
    if (cur_parity >= 0 && (((w0 & 1) != 0) != (cur_parity != 0)) && p.p_lo >= back) p.p_lo -= back;
    const long long range = p.p_hi - p.p_lo, smax = g.span_max & ~3;
    const long long nt = (range + smax - 1) / smax;
    p.n_tiles = (int) nt;
    p.span = nt > 0 ? (int) (((range + nt - 1) / nt + 3) & ~3LL) : 4;
}

int fused_smem_bytes(int bank_doubles_in_smem)
{
    return 2 * FPL * (int) sizeof(double2) + (256 + 256) * (int) sizeof(double2) + bank_doubles_in_smem * (int) sizeof(double);
}

int fused_poly_queue_bytes() { return POLY_QUEUE * (int) sizeof(int); }

int fused_poly_smem_bytes(int poly_dir, int poly_rows_cap, int poly_row_stride)
{
    return fused_smem_bytes(0) +
           (poly_dir != 0 ? poly_rows_cap * poly_row_stride * (int) sizeof(double) + fused_poly_queue_bytes() : 0);
}

PolyKnobs poly_knobs_env()
{
    PolyKnobs k;
    k.bank_global = getenv("R8BGPU_BANK_GLOBAL") != nullptr;
    k.single = getenv("R8BGPU_POLY_SINGLE") != nullptr;
    return k;
}

PolyCall plan_poly_call(const StageDesc& f, const FusedGeom& g, bool f2_poly, double ssr, double dsr, long long p_lo,
                        long long p_hi, int cur_parity, const PolyKnobs& k)
{
    PolyCall c;
    const double ratio = ssr / dsr;
    // order-2 bank on the v2 kernel: ratios within 1e-3 of an integer 1..3 (windows of consecutive outputs N apart)
    if (f2_poly) {
        const long long nn = llround(ratio);
        c.v2 = nn >= 1 && nn <= 3 && fabs(ratio - (double) nn) < 1e-3 * (double) nn;
        if (c.v2) c.poly_n = (int) nn;
    }
    if (c.v2) { // plain y layout, no staged rows
        FusedParams p;
        memset(&p, 0, sizeof p);
        p.p_lo = p_lo;
        p.p_hi = p_hi;
        fused2_tiles(p, g, cur_parity);
        c.n_tiles = p.n_tiles;
        c.span = p.span;
        c.p_lo = p.p_lo;
        return c;
    }
    // tile pairs: an even number of tiles of at most span_max positions (one tile alone when it covers the call)
    const long long range = p_hi - p_lo;
    long long nt = (range + g.span_max - 1) / g.span_max;
    if (nt > 1 && (nt & 1)) nt++;
    c.n_tiles = (int) nt;
    c.span = (int) (((range + nt - 1) / nt + 1) & ~1LL);
    c.p_lo = p_lo;
    c.ysh = g.ysh;
    const int flen = f.bank.filter_len;
    if ((flen & 1) == 0 && !k.bank_global) {
        // bank-row drift per output, in rows: frac(ssr/dsr) * fracs upward, or (1 - frac) * fracs downward
        const double fr = ratio - floor(ratio);
        const double outs = 2.0 * c.span / ratio + 4.0; // outputs one tile pair can own
        const int row_words = 6 * flen; // 32-bit words per bank row
        c.poly_row_stride = 3 * flen + ((row_words % 8) == 4 ? 0 : 2);
        const int cap = (224 * 1024 - fused_smem_bytes(0) - fused_poly_queue_bytes()) / (c.poly_row_stride * (int) sizeof(double));
        const double up = fr * f.bank.fracs * outs + 4.0, dn = (1.0 - fr) * f.bank.fracs * outs + 4.0;
        const double need = up < dn ? up : dn;
        const int chunks = (int) ceil(need / cap);
        if (cap >= 8 && chunks <= 4) { // more pieces than that: the rows are not a short run, read them from L2
            c.poly_dir = up < dn ? 1 : -1;
            c.poly_rows_cap = cap;
            c.poly_chunks = chunks < 1 ? 1 : chunks;
            const long long nn = llround(ratio);
            if (nn >= 1 && nn <= 3 && !k.single) {
                // four consecutive outputs per thread: lanes step by 4*nn samples through the tile -> padded
                // y layout (i + (i >> 4), the only padding the tile buffers have room for)
                c.poly_n = (int) nn;
                c.ysh = 4;
            }
        }
    }
    c.smem_bytes = fused_poly_smem_bytes(c.poly_dir, c.poly_rows_cap, c.poly_row_stride);
    return c;
}

int fused2_choose_glog(int span, int in_step, int out_step, int ir)
{
    // lanes = (32 >> glog) stepping cycles x (1 << glog) phase groups, 3 cycles per lane: fewest rounds of tasks
    // over a half-CTA's 8 warps, ties to the wider cycle dimension
    const int cyc = span / in_step + 2, ng = (out_step + ir - 1) / ir;
    int best = 0, best_rounds = INT_MAX;
    for (int gl = 0; gl <= 2; gl++) {
        const int tasks = ((ng + (1 << gl) - 1) >> gl) * ((cyc + (96 >> gl) - 1) / (96 >> gl));
        const int rounds = (tasks + 7) / 8;
        if (rounds < best_rounds) {
            best_rounds = rounds;
            best = gl;
        }
    }
    if (const char* e = getenv("R8BGPU_F2_GLOG")) best = atoi(e) & 3;
    return best > 2 ? 2 : best;
}

int fused2_choose_mbu(int span, int in_step, int out_step)
{
    // A tile owns ~span / in_step + 1 stepping cycles, handled in M tiles of 16 (pairs of 8-cycle blocks); a unit takes
    // 1..3 of them for one phase group.  Fewest (rounds over 8 warps) x (cost of a unit), where a unit's M tiles are
    // independent DMMA chains and fewer of them leave latency exposed: tools/mb_dmma.cu measured 0.55 / 0.41 / 0.38 clk per
    // output for 1 / 2 / 3 M tiles per unit (H100 80GB HBM3, 400 W).  Returns blocks (2 per M tile).
    static const int tile_cost[4] = {0, 143, 107, 100};
    const int cycles = span / in_step + 2, n_mt = (cycles - 1) / 16 + 1, n_groups = (out_step + 7) / 8;
    int best = 3;
    long long best_cost = LLONG_MAX;
    for (int mt = 3; mt >= 1; mt--) {
        const int units = n_groups * ((n_mt + mt - 1) / mt);
        const long long cost = (long long) ((units + 7) / 8) * mt * tile_cost[mt];
        if (cost < best_cost) {
            best_cost = cost;
            best = mt;
        }
    }
    best *= 2;
    if (const char* e = getenv("R8BGPU_F2_MBU")) best = atoi(e) & ~1;
    return best < 2 ? 2 : (best > f2::MBU_MAX ? f2::MBU_MAX : best);
}

} // namespace r8bgpu

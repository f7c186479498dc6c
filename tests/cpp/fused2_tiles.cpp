// Host check of the v2 fused kernel's per-call tile table (csrc/r8b_fused2_core.cuh, TileEntry / tile_entry): for
// every tile index of a call, the entry the kernel's prologue computes once must equal what each tile of each channel
// would compute for itself (interp_prepare on tile_of(u), or the order-2 bank's first outputs), for linear and ring
// destinations.  Calls are laid out by the engine's own host code (plan, schedule, tile geometry), the way
// r8b_capi.cu sets up k_up2_frac2.  TEST INFRASTRUCTURE: never linked into libr8bgpu.so.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../r8brain-free-src_b200/csrc/r8b_fused2_core.cuh"
#include "../../r8brain-free-src_b200/csrc/r8b_hosttab.h"
#include "../../r8brain-free-src_b200/csrc/r8b_plan.h"

using namespace r8bgpu;
using namespace r8bgpu::f2;

namespace {

// FusedParams of the pair (stage i, interpolator i + 1) for one call, as r8b_capi.cu fills the fields the tile
// bookkeeping reads
bool pair_params(const Plan& P, int i, const FusedGeom& g, const std::vector<StageCall>& calls, FusedParams& p)
{
    const StageDesc& f = P.stages[(size_t) i + 1];
    const StageCall& c = calls[(size_t) i];
    const StageCall& fc = calls[(size_t) i + 1];
    memset(&p, 0, sizeof p);
    if (f.kind == ST_FRAC_WHOLE) {
        fused_whole_fields(p, f, fc.e0, fc.e1);
    } else {
        p.mode = 1;
        p.flen = f.bank.filter_len;
        p.fll = p.flen / 2 - 1;
        p.e0 = fc.e0;
        p.e1 = fc.e1;
        p.p_lo = fc.p0 & ~1LL;
        p.p_hi = fc.p_last + 1;
        p.in_step = f.in_step;
        p.out_step = f.out_step;
        p.ssr = fc.ssr;
        p.dsr = fc.dsr;
        p.in_counter0 = fc.in_counter0;
        p.in_pos_int0 = fc.in_pos_int0;
        p.in_pos_shift = fc.in_pos_shift;
        p.fpos0 = fc.fpos0;
        p.p0 = fc.p0;
    }
    fused2_tiles(p, g, i == 0 ? (int) (c.n0 & 1) : -1);
    p.yl = g.yl;
    p.lg = g.lg;
    p.up = g.up;
    return fc.e1 > fc.e0;
}

// first k in [0, nk] whose read position is >= lim, by walking every output
long long poly_first_k_scan(const FusedParams& p, long long lim, long long nk)
{
    for (long long k = 0; k < nk; k++) {
        long long ip;
        double f;
        poly_position(p, k, ip, f);
        if (ip >= lim) return k;
    }
    return nk;
}

int g_reported = 0;
void report(const char* what, int call, int ti, int ch, long long got, long long want)
{
    if (g_reported++ < 8)
        fprintf(stderr, "tile table mismatch (%s): call %d tile %d channel %d: %lld, per tile %lld\n", what, call, ti, ch, got, want);
}

} // namespace

extern "C" {

// Runs a stream of calls of the given lengths through every fused pair of the plan.  stats: [0] entries checked,
// [1] whole-stepping pairs, [2] order-2 bank pairs, [3] calls whose first tile reaches before the caller's block
// (into the history ring), [4] largest tile count of a call.  Returns the number of mismatches, -1 without a fused pair.
int f2tiles_check(double src, double dst, int max_len, double tb, double atten, const int* lens, int n_lens, long long* stats)
{
    Plan P;
    if (!P.build(src, dst, max_len, tb, atten, 0, 0, 0)) return -1;
    std::vector<int> pairs;
    std::vector<FusedGeom> geoms;
    for (size_t i = 0; i + 1 < P.stages.size(); i++) {
        const FusedGeom g = fused_geometry(P.stages[i], P.stages[i + 1]);
        if (g.ok) {
            pairs.push_back((int) i);
            geoms.push_back(g);
        }
    }
    if (pairs.empty()) return -1;
    for (size_t k = 0; k < pairs.size(); k++) stats[P.stages[(size_t) pairs[k] + 1].kind == ST_FRAC_WHOLE ? 1 : 2]++;
    Schedule S;
    S.init(&P);
    std::vector<StageCall> calls;
    int bad = 0;
    static double dummy[1];
    for (int call = 0; call < n_lens; call++) {
        S.advance(lens[call], calls);
        for (size_t k = 0; k < pairs.size(); k++) {
            const int i = pairs[k];
            FusedParams p;
            if (!pair_params(P, i, geoms[k], calls, p)) continue;
            if (p.n_tiles > stats[4]) stats[4] = p.n_tiles;
            if (i == 0 && tile_of(p, 0).w < calls[0].n0) stats[3]++;
            const long long nk = p.e1 - p.e0;
            long long ja_next = p.e0;
            for (int ti = 0; ti < p.n_tiles; ti++) {
                // the entry as the kernel's prologue computes it, for a destination whose element 0 is output e0
                const TileEntry e = tile_entry(p, p.e0, ti);
                stats[0]++;
                if (p.mode == 1) {
                    const Tile t = tile_of(p, ti);
                    const long long ka = poly_first_k_scan(p, t.A0, nk), kb = poly_first_k_scan(p, t.A1, nk);
                    if (e.s[0] != ka) report("first output", call, ti, 0, e.s[0], ka), bad++;
                    if (e.s[1] != kb) report("end output", call, ti, 0, e.s[1], kb), bad++;
                    continue;
                }
                // the tiles' outputs [ja, ja + n) follow one another and cover the call
                if (e.s[0] > 0) {
                    if (p.e0 + e.off != ja_next) report("first output", call, ti, 0, p.e0 + e.off, ja_next), bad++;
                    ja_next = p.e0 + e.off + e.s[0];
                }
                // every channel's tile of this index, linear (base e0, row stride 1e6 + 3) and ring (base 0, 2^18) rows
                for (int ch : {0, 1, 7, 2999}) {
                    for (int ring = 0; ring < 2; ring++) {
                        DstView d;
                        d.ptr = dummy;
                        d.stride = ring ? (1LL << 18) : 1000003LL;
                        d.mask = ring ? (1LL << 18) - 1 : -1;
                        d.base = ring ? 0 : p.e0;
                        const TileEntry er = ring ? tile_entry(p, 0, ti) : e;
                        const Tile t = tile_of(p, ch * p.n_tiles + ti);
                        int s_i[8];
                        double* s_o = nullptr;
                        interp_prepare(p, d, t, s_i, &s_o);
                        for (int j = 0; j < 4; j++)
                            if (er.s[j] != s_i[j]) report("s_i", call, ti, ch, er.s[j], s_i[j]), bad++;
                        const long long row = (long long) ch * d.stride;
                        if (s_o - d.ptr != row + (er.off & d.mask)) report("slot", call, ti, ch, row + (er.off & d.mask), s_o - d.ptr), bad++;
                        MmaTile a, b;
                        a.load(er, row);
                        b.load(s_i);
                        if (!ring && a.elem0 != b.elem0) report("element", call, ti, ch, a.elem0, b.elem0), bad++;
                    }
                }
            }
            if (p.mode == 0 && ja_next != p.e1) report("outputs covered", call, -1, 0, ja_next, p.e1), bad++;
        }
    }
    return bad;
}

} // extern "C"

// Host replay of k_up2_frac's order-2 bookkeeping (csrc/r8b_fused.cu, mode 1): for every call of a stream, the call's
// decision (plan_poly_call, the function r8b_capi.cu launches from), then every tile pair's outputs [ka, kb), its chunks,
// their staged bank rows, and each output's bank row and window -- with the very functions the kernel runs
// (r8b_poly.cuh).  Checks that the pairs' ranges partition the call's outputs and each pair owns exactly the outputs
// whose read position lies in its tiles, that every owned window lies inside its tile buffer (PolyOut::ok) and inside the
// part of the tile the overlap-save transform makes valid, and that every staged row read is the bank row it stands for.
// Counts what a sweep must reach (directions, chunk counts, wrapped and whole-bank runs, the deferred-output queue).
// TEST INFRASTRUCTURE: never linked into libr8bgpu.so.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../r8brain-free-src_b200/csrc/r8b_fused2_core.cuh"
#include "../../r8brain-free-src_b200/csrc/r8b_hosttab.h"
#include "../../r8brain-free-src_b200/csrc/r8b_plan.h"

using namespace r8bgpu;

namespace {

// stats[] indices (tests/test_order2_geometry_cpu.py names them)
enum {
    S_CALLS,        // calls that launch the pair
    S_PAIRS,        // tile pairs (CTAs of one channel)
    S_OUTPUTS,      // outputs replayed
    S_BAD_OWN,      // pair ranges that do not partition the call, or outputs owned by the wrong pair
    S_NOT_OK,       // owned outputs whose window leaves the tile buffer (skipped by the kernel)
    S_BAD_ROW,      // staged rows that are not the bank row read through them, or runs past the staging area
    S_NOT_VALID,    // owned windows reaching outside the tile's valid (overlap-save) samples
    S_MAX_QUEUE,    // most outputs one chunk defers to the one-output-per-lane pass
    S_OVERFLOW,     // chunks that defer more than POLY_QUEUE outputs
    S_ROW_FRACS,    // outputs whose bank row is row `fracs` (the extra row; read from global memory)
    S_MAX_NST,      // longest staged run
    S_WHOLE_BANK,   // chunks that stage the whole bank (n_st == fracs)
    S_WRAP_UP,      // chunks whose staged run wraps past row fracs - 1, rows ascending
    S_WRAP_DN,      // ... rows descending
    S_MAX_CHUNKS,   // most chunks of a call
    S_FAST,         // outputs computed by poly_block4 (four per thread, one staged row)
    S_ODD_TILES,    // calls whose last pair has no tile b
    S_DIR_UP,       // calls staging ascending runs
    S_DIR_DN,       // calls staging descending runs
    S_DIR_NONE,     // calls staging nothing
    S_STAGED_READS, // outputs reading a staged row
    S_FT_CALLS,     // calls on R8B_FASTTIMING position tables
    S_ROW0_WRAP,    // chunks whose first row is row 0, so the run starts at fracs - 1
    S_DIR_FLIPS,    // consecutive launching calls whose staging direction flips between +1 and -1
    S_V2_CALLS,     // calls that run on k_up2_frac2<POLY> (R8BGPU_POLY_V2; its tiles are not replayed here)
    S_N
};
// per-call fields: range, n_tiles, span, dir, rows, stride, chunks, n, ysh, queue peak, launched, on k_up2_frac2 (not
// replayed), chunks whose run starts at row fracs - 1 because their first row is 0, highest bank row read
constexpr int PC_N = 14;

int g_reported = 0;
void report(const char* what, int call, int pair, long long k, long long a, long long b)
{
    if (g_reported++ < 10)
        fprintf(stderr, "order2 pairs: %s: call %d pair %d output %lld: %lld vs %lld\n", what, call, pair, k, a, b);
}

} // namespace

extern "C" {

// kind 0: Plan::build(src, dst, max_len, tb, atten, fasttiming); 1: build_trim; 2: build_trim(any_pair).  Call c feeds
// lens[c] samples after setting the trim factor factors[c] (trim plans).  f2_poly: the plan may run the pair on
// k_up2_frac2 (FusedPlan::poly_v2: R8BGPU_POLY_V2 on a plan that meets plan_fused_stage's conditions); calls that do
// are counted, not replayed.  Returns -1 when the plan has no fused order-2
// pair, else the sum of the failure counts (stats[S_BAD_OWN] + S_NOT_OK + S_BAD_ROW + S_NOT_VALID).
int o2pairs_run(int kind, double src, double dst, int max_len, double tb, double atten, int fasttiming, double max_trim,
                const int* lens, const double* factors, int n_calls, int bank_global, int single, int f2_poly,
                long long* stats,
                long long* per_call)
{
    Plan P;
    const bool ok = kind == 0 ? P.build(src, dst, max_len, tb, atten, 0, 0, fasttiming)
                              : P.build_trim(src, dst, max_len, tb, atten, 0, max_trim, kind == 2);
    if (!ok) return -1;
    int pi = -1;
    FusedGeom g;
    for (size_t i = 0; i + 1 < P.stages.size(); i++) {
        if (P.stages[i + 1].kind != ST_FRAC_POLY) continue;
        g = fused_geometry(P.stages[i], P.stages[i + 1]);
        if (g.ok) pi = (int) i;
    }
    if (pi < 0) return -1;
    const StageDesc& f = P.stages[(size_t) pi + 1];
    PolyKnobs knobs;
    knobs.bank_global = bank_global != 0;
    knobs.single = single != 0;
    memset(stats, 0, S_N * sizeof(long long));
    Schedule S;
    S.init(&P);
    std::vector<StageCall> calls;
    int last_dir = 0;
    for (int call = 0; call < n_calls; call++) {
        long long* pc_out = per_call + (size_t) call * PC_N;
        memset(pc_out, 0, PC_N * sizeof(long long));
        if (P.trim_stage >= 0) S.retime(P.trim_dsr(factors[call]));
        S.advance(lens[call], calls);
        const StageCall& fc = calls[(size_t) pi + 1];
        if (fc.e1 <= fc.e0) continue;
        // the fields launch_call fills for the pair
        FusedParams p;
        memset(&p, 0, sizeof p);
        p.mode = 1;
        p.flen = f.bank.filter_len;
        p.fll = p.flen / 2 - 1;
        p.e0 = fc.e0;
        p.e1 = fc.e1;
        p.p_lo = fc.p0 & ~1LL;
        p.p_hi = fc.p_last + 1;
        p.in_step = f.in_step;
        p.out_step = f.out_step;
        p.fracs = f.bank.fracs;
        p.ssr = fc.ssr;
        p.dsr = fc.dsr;
        p.in_counter0 = fc.in_counter0;
        p.in_pos_int0 = fc.in_pos_int0;
        p.in_pos_shift = fc.in_pos_shift;
        p.fpos0 = fc.fpos0;
        p.p0 = fc.p0;
        p.bank = f.bank.table.data();
        if (!fc.ft_dp.empty()) {
            p.pos_dp = fc.ft_dp.data();
            p.pos_fpos = fc.ft_fpos.data();
            stats[S_FT_CALLS]++;
        }
        const PolyCall pc = plan_poly_call(f, g, f2_poly != 0, fc.ssr, fc.dsr, p.p_lo, p.p_hi, -1, knobs);
        if (pc.v2) {
            pc_out[0] = p.p_hi - p.p_lo;
            pc_out[10] = 1;
            pc_out[11] = 1;
            stats[S_V2_CALLS]++;
            continue;
        }
        p.n_tiles = pc.n_tiles;
        p.span = pc.span;
        p.p_lo = pc.p_lo;
        p.yl = g.yl;
        p.lg = g.lg;
        p.ysh = pc.ysh;
        p.poly_dir = pc.poly_dir;
        p.poly_rows_cap = pc.poly_rows_cap;
        p.poly_row_stride = pc.poly_row_stride;
        p.poly_chunks = pc.poly_chunks;
        p.poly_n = pc.poly_n;
        const long long pcv[9] = {p.p_hi - p.p_lo, p.n_tiles, p.span, p.poly_dir, p.poly_rows_cap, p.poly_row_stride,
                                  p.poly_chunks, p.poly_n, p.ysh};
        for (int j = 0; j < 9; j++) pc_out[j] = pcv[j];
        pc_out[10] = 1;
        stats[S_CALLS]++;
        stats[p.poly_dir > 0 ? S_DIR_UP : p.poly_dir < 0 ? S_DIR_DN : S_DIR_NONE]++;
        if (p.poly_dir != 0 && last_dir != 0 && p.poly_dir != last_dir) stats[S_DIR_FLIPS]++;
        if (p.poly_dir != 0) last_dir = p.poly_dir;
        if (p.n_tiles & 1) stats[S_ODD_TILES]++;
        if (p.poly_chunks > stats[S_MAX_CHUNKS]) stats[S_MAX_CHUNKS] = p.poly_chunks;
        // the staged rows and the queue fit the launch's dynamic shared memory
        if (p.poly_dir != 0 && (p.poly_row_stride < 3 * p.flen || pc.smem_bytes > 224 * 1024)) stats[S_BAD_ROW]++;
        const long long nk = p.e1 - p.e0;
        const int n_pairs = (p.n_tiles + 1) >> 1;
        long long k_next = 0;
        for (int pair = 0; pair < n_pairs; pair++) {
            stats[S_PAIRS]++;
            // k_up2_frac's prologue, as written there
            const int ta = 2 * pair;
            const bool has_b = (ta + 1) < p.n_tiles;
            const long long A0 = p.p_lo + (long long) ta * p.span;
            long long A1 = A0 + p.span;
            if (A1 > p.p_hi) A1 = p.p_hi;
            const long long B0 = A1;
            long long B1 = has_b ? B0 + p.span : B0;
            if (B1 > p.p_hi) B1 = p.p_hi;
            const long long wa = (A0 - p.yl) / 2 - p.lg, wb = (B0 - p.yl) / 2 - p.lg;
            const long long ya0 = 2 * wa, yb0 = 2 * wb;
            const long long bsel = has_b ? B0 - p.yl : LLONG_MAX;
            const long long ka = poly_first_k(p, A0, nk), kb = poly_first_k(p, B1, nk);
            if (ka != k_next) report("pair starts off the previous pair's end", call, pair, ka, ka, k_next), stats[S_BAD_OWN]++;
            k_next = kb;
            for (int c = 0; c < p.poly_chunks; c++) {
                const long long k_lo = poly_chunk_start(ka, kb, c, p.poly_chunks), k_hi = poly_chunk_start(ka, kb, c + 1, p.poly_chunks);
                int r_lo, n_st;
                poly_rows_for(p, k_lo, k_hi, r_lo, n_st);
                if (n_st > 0) {
                    if (n_st > p.poly_rows_cap || n_st > p.fracs || r_lo < 0 || r_lo >= p.fracs)
                        report("staged run", call, pair, k_lo, r_lo, n_st), stats[S_BAD_ROW]++;
                    if (n_st > stats[S_MAX_NST]) stats[S_MAX_NST] = n_st;
                    if (n_st == p.fracs) stats[S_WHOLE_BANK]++;
                    if (r_lo + n_st > p.fracs) stats[p.poly_dir > 0 ? S_WRAP_UP : S_WRAP_DN]++;
                    if (r_lo == p.fracs - 1) {
                        stats[S_ROW0_WRAP]++;
                        pc_out[12]++;
                    }
                }
                // poly_stage_rows: slot sl holds row (r_lo + sl) mod fracs
                auto staged_row = [&](int sl) {
                    int row = r_lo + sl;
                    if (row >= p.fracs) row -= p.fracs;
                    return row;
                };
                long long queued = 0;
                const int NN = p.poly_n > 0 ? p.poly_n : 1;
                auto check_out = [&](const PolyOut& o, long long k) {
                    stats[S_OUTPUTS]++;
                    long long ip;
                    double fpos;
                    poly_position(p, k, ip, fpos);
                    if (ip < A0 || ip >= B1) report("output owned by another pair", call, pair, k, ip, A0), stats[S_BAD_OWN]++;
                    if (!o.ok) report("window outside the tile buffer", call, pair, k, o.yi, 2 * FM), stats[S_NOT_OK]++;
                    // valid samples of a tile: local input-rate indices [lg, FM - lg) of its transform window
                    if (o.yi < 2 * p.lg || o.yi + p.flen > 2 * (FM - p.lg))
                        report("window outside the valid samples", call, pair, k, o.yi, 2 * p.lg), stats[S_NOT_VALID]++;
                    if (o.fti >= p.fracs) stats[S_ROW_FRACS]++;
                    if (o.fti > pc_out[13]) pc_out[13] = o.fti;
                    if (o.fti < 0 || o.fti > p.fracs) report("bank row", call, pair, k, o.fti, p.fracs), stats[S_BAD_ROW]++;
                    const int slot = poly_slot(p, r_lo, o.fti);
                    if (slot < n_st && o.fti < p.fracs) { // poly_single reads the staged row
                        stats[S_STAGED_READS]++;
                        if (staged_row(slot) != o.fti) report("staged row", call, pair, k, staged_row(slot), o.fti), stats[S_BAD_ROW]++;
                    }
                };
                if (p.poly_n == 0) {
                    for (long long k = k_lo; k < k_hi; k++) check_out(poly_output(p, ya0, yb0, bsel, k), k);
                } else {
                    for (long long k = k_lo; k < k_hi; k += 4) {
                        PolyOut o[4];
                        const int nv = (int) (k_hi - k < 4 ? k_hi - k : 4);
                        for (int r = 0; r < nv; r++) o[r] = poly_output(p, ya0, yb0, bsel, k + r);
                        int slot;
                        const bool fast = NN == 1 ? poly_fast_group<1>(p, o, nv, r_lo, n_st, slot)
                                        : NN == 2 ? poly_fast_group<2>(p, o, nv, r_lo, n_st, slot)
                                                  : poly_fast_group<3>(p, o, nv, r_lo, n_st, slot);
                        for (int r = 0; r < nv; r++) check_out(o[r], k + r);
                        if (fast) {
                            stats[S_FAST] += 4;
                            if (staged_row(slot) != o[0].fti) report("block row", call, pair, k, staged_row(slot), o[0].fti), stats[S_BAD_ROW]++;
                        } else {
                            queued += nv;
                        }
                    }
                }
                if (queued > stats[S_MAX_QUEUE]) stats[S_MAX_QUEUE] = queued;
                if (queued > pc_out[9]) pc_out[9] = queued;
                if (queued > POLY_QUEUE) stats[S_OVERFLOW]++;
            }
        }
        if (k_next != nk) report("pairs end before the call's last output", call, -1, k_next, k_next, nk), stats[S_BAD_OWN]++;
    }
    return (int) (stats[S_BAD_OWN] + stats[S_NOT_OK] + stats[S_BAD_ROW] + stats[S_NOT_VALID]);
}

// poly_first_k(lim) for a call whose timing state is (in_counter0 c0, in_pos_shift, in_pos_int0 int0, p0) at rates
// ssr / dsr, and the same first output found by walking every output with poly_position: *scan.
long long o2first_k(double ssr, double dsr, double shift, int c0, int int0, long long p0, long long lim, long long nk,
                    long long* scan)
{
    FusedParams p;
    memset(&p, 0, sizeof p);
    p.ssr = ssr;
    p.dsr = dsr;
    p.in_pos_shift = shift;
    p.in_counter0 = c0;
    p.in_pos_int0 = int0;
    p.p0 = p0;
    *scan = nk;
    for (long long k = 0; k < nk; k++) {
        long long ip;
        double f;
        poly_position(p, k, ip, f);
        if (ip >= lim) {
            *scan = k;
            break;
        }
    }
    return poly_first_k(p, lim, nk);
}

} // extern "C"

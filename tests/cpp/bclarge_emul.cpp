// CPU emulation of the large-tile BlockConvolver (k_bcl_gather, k_bcl_conv, k_bcl_scatter; csrc/r8b_bclarge.cuh), for
// the tests that run without a GPU.
//
// The kernels' per-thread steps compile for the host.  This harness runs them "thread" after "thread", one loop per
// kernel (and per barrier interval inside k_bcl_conv), on a one-stage plan of the engine (Plan::build_single) with its
// own schedule, tile choice, per-call tile geometry and spectrum tables, so the radix-R0 split, the slot order, the
// Nyquist injection and the scatter bookkeeping are checked against the reference's own stage before a GPU is
// involved.  It also exposes the host tile choice for every BlockConvolver stage of a whole plan.
// TEST INFRASTRUCTURE: not part of the product, never linked into libr8bgpu.so.
#include <chrono>
#include <cstring>
#include <vector>

#include "../../r8brain-free-src_b200/csrc/r8b_bclarge.cuh"
#include "../../r8brain-free-src_b200/csrc/r8b_hosttab.h"
#include "../../r8brain-free-src_b200/csrc/r8b_plan.h"

using namespace r8bgpu;

namespace {

struct Emul {
    Plan plan;
    Schedule sched;
    std::vector<StageCall> calls;
    BcTile tile;
    std::vector<double2> spec, tw4096, tw_m, scratch;
    double nyq_gain = 0.0;
    std::vector<double> ring; // the whole past of the input stream (power-of-two ring, zero before the start)
    long long ring_mask = 0;
    double spectrum_ms = 0.0;
};

// k_bcl_conv for one (unit, sub-block): the block-wide passes of fft_forward / fft_inverse<4096> (r8b_fft.cuh) run
// butterfly after butterfly
void conv_block(const BcLargeParams& p, double2* blk, int r)
{
    using namespace bcl;
    std::vector<double2> sm((size_t) SUB_PL);
    double2* s = sm.data();
    const double2* tw = p.bc.tw;
    for (int n = 0; n < SUB; n++) s[fft_pad(n)] = blk[n];
    for (int g = 0; g < SUB / 16; g++) fft_bfly_forward<SUB, SUB, 16>(s, tw, g);
    for (int g = 0; g < SUB / 16; g++) fft_bfly_forward<SUB, 256, 16>(s, tw, g);
    for (int g = 0; g < SUB / 16; g++) fft_bfly_forward<SUB, 16, 16>(s, tw, g);
    const bool nyq_here = p.bc.trunc > 0 && r == 0;
    const double2 nyq = nyq_here ? conv_nyquist(p, s) : make_double2(0.0, 0.0);
    for (int k = 0; k < SUB; k++) conv_mul_item(p, s, r, k, nyq_here, nyq);
    for (int g = 0; g < SUB / 16; g++) fft_bfly_inverse<SUB, 16, 16>(s, tw, g);
    for (int g = 0; g < SUB / 16; g++) fft_bfly_inverse<SUB, 256, 16>(s, tw, g);
    for (int g = 0; g < SUB / 16; g++) fft_bfly_inverse<SUB, SUB, 16>(s, tw, g);
    for (int n = 0; n < SUB; n++) blk[n] = s[fft_pad(n)];
}

template <int R0>
void run_call(const BcLargeParams& p, const SrcView& src, const DstView& dst, int n_units)
{
    using namespace bcl;
    for (int u = 0; u < n_units; u++) {
        const Pair t = pair_of(p.bc, u);
        for (int n1 = 0; n1 < SUB; n1++) gather_item<R0>(p, src, t, n1, p.scratch + (size_t) u * R0 * SUB);
    }
    for (int b = 0; b < n_units * R0; b++) conv_block(p, p.scratch + (size_t) b * SUB, b % R0);
    for (int u = 0; u < n_units; u++) {
        const Pair t = pair_of(p.bc, u);
        for (int n1 = 0; n1 < SUB; n1++) scatter_item<R0>(p, dst, t, n1, p.scratch + (size_t) u * R0 * SUB);
    }
}

} // namespace

extern "C" {

// Host tile choice of every BlockConvolver stage of the plan (src, dst, ...): 10 ints per stage -- up, down,
// block_exact, half_len, ref_prev_len, block_len_bits + 1, then the choice: fft_log2, large, lg, virt_up.  Returns the
// number of BlockConvolver stages, -1 when the plan is refused.
int bclemul_tiles(double src, double dst, int max_in, double tb, double atten, int extfft, int* out, int cap)
{
    Plan P;
    if (!P.build(src, dst, max_in, tb, atten, 0, extfft, 0)) return -1;
    int n = 0;
    for (const StageDesc& s : P.stages) {
        if (s.kind != ST_BLOCKCONV) continue;
        if (n < cap) {
            const BcTile t = blockconv_tile(s);
            int* o = out + 10 * n;
            o[0] = s.up;
            o[1] = s.down;
            o[2] = s.block_exact ? 1 : 0;
            o[3] = s.lp.half_len;
            o[4] = s.ref_prev_len;
            o[5] = s.lp.block_len_bits + 1;
            o[6] = t.fft_log2;
            o[7] = t.large ? 1 : 0;
            o[8] = t.lg;
            o[9] = t.virt_up;
        }
        n++;
    }
    return n;
}

// The first BlockConvolver stage of the plan (src, dst, ...) that takes the large-tile path: a[0..5] = {norm_freq,
// trans_band, atten, gain, up, down} (Plan::build_single / the reference's stage), returns its longest input per call
// (-1: no such stage).
int bclemul_find(double src, double dst, int max_in, double tb, double atten, int extfft, double* a)
{
    Plan P;
    if (!P.build(src, dst, max_in, tb, atten, 0, extfft, 0)) return -1;
    int in_len = max_in;
    for (const StageDesc& s : P.stages) {
        if (s.kind == ST_BLOCKCONV && blockconv_tile(s).large) {
            a[0] = s.norm_freq;
            a[1] = s.trans_band;
            a[2] = P.atten;
            a[3] = s.gain;
            a[4] = s.up;
            a[5] = s.down;
            return in_len;
        }
        in_len = s.max_out_len;
    }
    return -1;
}

// One large-tile BlockConvolver stage for ONE channel; NULL when the stage does not take the large-tile path.
void* bclemul_create(const double* a, int max_in, int extfft)
{
    Emul* E = new Emul;
    if (!E->plan.build_single(ST_BLOCKCONV, a, max_in, extfft) || E->plan.stages.size() != 1) {
        delete E;
        return nullptr;
    }
    const StageDesc& s = E->plan.stages[0];
    E->tile = blockconv_tile(s);
    if (!E->tile.large) {
        delete E;
        return nullptr;
    }
    const auto t0 = std::chrono::steady_clock::now();
    build_spectrum_large(s, E->tile.fft_log2, E->spec, E->tw4096, E->tw_m, &E->nyq_gain);
    E->spectrum_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    E->sched.init(&E->plan);
    E->ring.assign((size_t) 1 << 22, 0.0);
    E->ring_mask = ((long long) 1 << 22) - 1;
    return E;
}

void bclemul_destroy(void* h) { delete (Emul*) h; }

// info[0..3] = fft_log2, lg, virt_up, block_exact; returns the milliseconds build_spectrum_large took
double bclemul_info(void* h, int* info)
{
    const Emul& E = *(const Emul*) h;
    info[0] = E.tile.fft_log2;
    info[1] = E.tile.lg;
    info[2] = E.tile.virt_up;
    info[3] = E.plan.stages[0].block_exact ? 1 : 0;
    return E.spectrum_ms;
}

// One process() call: l input samples at x, up to out_cap outputs; returns the count.
int bclemul_process(void* h, const double* x, int l, double* out, int out_cap)
{
    Emul& E = *(Emul*) h;
    const int n_out = E.sched.advance(l, E.calls);
    if (n_out > out_cap) return -1;
    const StageCall& c = E.calls[0];
    const StageDesc& s = E.plan.stages[0];
    if (c.e1 > c.e0) {
        BcLargeParams p;
        blockconv_call_fields(p.bc, s, E.tile.virt_up, E.tile.lg, E.tile.fft_log2, c.e0, c.e1);
        p.bc.nyq_gain = E.nyq_gain;
        p.bc.spec = E.spec.data();
        p.bc.tw = E.tw4096.data();
        p.tw_m = E.tw_m.data();
        const int units = bcl::n_pairs(p.bc), M = 1 << E.tile.fft_log2;
        E.scratch.assign((size_t) units * M, make_double2(0.0, 0.0));
        p.scratch = E.scratch.data();
        p.group_ch = 1;
        SrcView src;
        src.ring = E.ring.data();
        src.ring_stride = (long long) E.ring.size();
        src.ring_mask = E.ring_mask;
        src.cur = x;
        src.cur_stride = l;
        src.cur_base = c.n0;
        src.avail = c.n1;
        DstView dst;
        dst.ptr = out;
        dst.stride = out_cap;
        dst.mask = -1;
        dst.base = c.e0;
        if (M == 16384) run_call<4>(p, src, dst, units);
        else if (M == 32768) run_call<8>(p, src, dst, units);
        else run_call<16>(p, src, dst, units);
    }
    for (int i = 0; i < l; i++) E.ring[(size_t) ((c.n0 + i) & E.ring_mask)] = x[i];
    return n_out;
}

} // extern "C"

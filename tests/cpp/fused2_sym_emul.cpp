// CPU emulation of the v2 fused kernel (csrc/r8b_fused2.cu) with phase C on the symmetric half-size spectrum table
// (FusedParams::cs_tab, cd1s_compute), for the tests that run without a GPU.
//
// The same driver as fused2_emul.cpp -- the kernel's per-thread phase functions (csrc/r8b_fused2_core.cuh) run "thread"
// after "thread", one loop per barrier interval, on tiles laid out by the engine's own host code -- except that the 2x
// pair's phase C reads the table the kernel keeps in shared memory.  Also exposed: the bins of G rebuilt from that table
// with the kernel's own arithmetic next to the full slot-ordered spectrum, and the per-plan shared-memory fit decision.
// TEST INFRASTRUCTURE: not part of the product, never linked into libr8bgpu.so.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../r8brain-free-src_b200/csrc/r8b_fused2_core.cuh"
#include "../../r8brain-free-src_b200/csrc/r8b_hosttab.h"
#include "../../r8brain-free-src_b200/csrc/r8b_plan.h"

using namespace r8bgpu;
using namespace r8bgpu::f2;

namespace {

struct Emul {
    Plan plan;
    Schedule sched;
    std::vector<StageCall> calls;
    FusedGeom fg;
    GroupBank B;
    std::vector<double2> spec, tw, tw_tab, c_tab, cs_tab;
    std::vector<double> ring; // the whole past of the input stream (power-of-two ring, zero before the start)
    long long ring_mask = 0;
    int glog_force = -1;
    bool tc = false; // interpolation through the m8n8k4 formulation (glog_force == 8)
};

// the tensor-path interpolation: one m8n8k4 product per (block of 8 cycles, K-step), emulated on whole "warps" with the
// fragment layouts of mma.sync (A: lane = 4*row + k, B: lane = 4*n + k, C: lane = 4*row + col/2)
template <bool PADV>
void interp_tc(const FusedParams& p, const DstView& dst, const Tile& t, const double* yb, const double* sbank, const int* s_goff,
               const int* s_i, double* s_o)
{
    MmaTile mt;
    mt.load(s_i);
    const int n_groups = (p.out_step + 7) / 8;
    const int n_mu = mma_units(p, mt.c_cnt), ksteps = p.smaxp >> 2;
    for (int w = 0; w < HT / 32; w++) { // the kernel deals units to its 8 warps round-robin
        MmaUnit mu;
        mu.set(w, n_groups);
        for (int unit = w; unit < n_mu; unit += HT / 32, mu.advance(HT / 32, n_groups)) {
            const int MBU = mma_mbu(p);
            double acc[MBU_MAX][32][2] = {};
            for (int ks = 0; ks < ksteps; ks++) {
                double b[32];
                for (int lane = 0; lane < 32; lane++) b[lane] = sbank[mma_b_index(p, mu, lane) + ks * 32];
                for (int i = 0; i < MBU; i++) {
                    double a[32];
                    for (int lane = 0; lane < 32; lane++) {
                        const int yi = mma_a_index(p, mt, mu, s_goff[mu.g], i, lane) + 4 * ks;
                        a[lane] = PADV ? yb[ylay(yi, p.ysh)] : yb[yi];
                    }
                    for (int lane = 0; lane < 32; lane++) {
                        const int row = lane >> 2, col = 2 * (lane & 3);
                        for (int k = 0; k < 4; k++) {
                            acc[i][lane][0] = fma(a[4 * row + k], b[4 * col + k], acc[i][lane][0]);
                            acc[i][lane][1] = fma(a[4 * row + k], b[4 * (col + 1) + k], acc[i][lane][1]);
                        }
                    }
                }
            }
            for (int i = 0; i < MBU; i++)
                for (int lane = 0; lane < 32; lane++) mma_store(p, dst, t.ch, mt, s_o, mu, i, lane, acc[i][lane][0], acc[i][lane][1]);
        }
    }
}

template <int IR, bool PADV, int GLOG>
void run_units(const FusedParams& p, const SrcView& src, const DstView& dst, const Emul& E)
{
    std::vector<double2> buf((size_t) FPL2);
    const double2* tw2 = E.tw_tab.data();
    const double2* twf = tw2 + 256;
    const int n_groups = (p.out_step + IR - 1) / IR, esz = p.smaxp * IR;
    // this call's bank selection, as the kernel's bulk copies lay it out
    std::vector<double> sbank((size_t) n_groups * esz);
    std::vector<int> s_goff((size_t) n_groups);
    for (int g = 0; g < n_groups; g++) {
        memcpy(&sbank[(size_t) g * esz], p.gbank + (long long) (p.delta + g * IR) * esz, (size_t) esz * sizeof(double));
        s_goff[(size_t) g] = p.goff[p.delta + g * IR];
    }
    const int n_units = p.n_tiles * p.n_ch;
    for (int u = 0; u < n_units; u++) {
        const Tile t = tile_of(p, u);
        const int path = tile_input_path(src, t);
        if (path == 2) // the bulk copy
            memcpy(buf.data() + fft_pad(FN), tile_run(src, t), FM * sizeof(double));
        for (int ht = 0; ht < HT; ht++) {
            double2 v[8];
            if (path == 2) {
                for (int j = 0; j < 8; j++) v[j] = buf[(size_t) (fft_pad(FN) + ht + 256 * j)];
            } else {
                gather_tile(v, src, t, path, ht);
            }
            fwd_pass1_r8(v, buf.data(), tw2, twf, ht);
        }
        int s_i[8];
        double* s_o = nullptr;
        interp_prepare(p, dst, t, s_i, &s_o);
        for (int ht = 0; ht < FN / 16; ht++) fwd_pass<256>(buf.data(), tw2, ht);
        if (p.up == 1) for (int ht = 0; ht < FN / 16; ht++) fwd_pass<16>(buf.data(), tw2, ht);
        else for (int ht = 0; ht < FN / 16; ht++) fwd_pass16_skew(buf.data(), ht);
        if (p.up == 1) {
            std::vector<double2> z1((size_t) HT * 4), z2((size_t) HT * 4);
            for (int ht = 0; ht < HT; ht++) {
                double2 a[4], b[4];
                c_load(buf.data(), ht, a, b);
                for (int i = 0; i < 4; i++) {
                    z1[(size_t) ht * 4 + i] = a[i];
                    z2[(size_t) ht * 4 + i] = b[i];
                }
            }
            const double2 ze = buf[(size_t) fft_pad(slot_of<FN>(FN / 2))];
            for (int ht = 0; ht < HT; ht++)
                for (int i = 0; i < 4; i++) c1_pair_tab(p, buf.data(), ht, i, z1[(size_t) ht * 4 + i], z2[(size_t) ht * 4 + i]);
            c1_pair_mid(p, buf.data(), ze);
        } else { // phase C inside the first inverse pass: every "thread" fetches, then (after the barrier) computes
            std::vector<double2> z1((size_t) HT * 8), z2((size_t) HT * 8);
            for (int ht = 0; ht < HT; ht++) {
                double2 a[8], b[8];
                cd1_load(buf.data(), ht, a, b);
                for (int i = 0; i < 8; i++) {
                    z1[(size_t) ht * 8 + i] = a[i];
                    z2[(size_t) ht * 8 + i] = b[i];
                }
            }
            const double2* cs = E.cs_tab.data(); // the kernel's shared-memory copy: the first CS_PAIRS entries
            for (int ht = 0; ht < HT; ht++) {
                double2 a[8], b[8];
                for (int i = 0; i < 8; i++) {
                    a[i] = z1[(size_t) ht * 8 + i];
                    b[i] = z2[(size_t) ht * 8 + i];
                }
                cd1s_compute(cs, cs[CS_PAIRS + ht], cs[CS_PAIRS + HT + ht], buf.data(), ht, a, b);
            }
        }
        if (p.up == 1) {
            for (int ht = 0; ht < FN / 16; ht++) inv_pass<16>(buf.data(), tw2, ht);
            for (int ht = 0; ht < FN / 16; ht++) inv_pass<256>(buf.data(), tw2, ht);
            std::vector<double2> v((size_t) HT * 8);
            for (int ht = 0; ht < HT; ht++) {
                double2 a[8];
                inv1_last_load(buf.data(), tw2, twf, ht, a);
                for (int i = 0; i < 8; i++) v[(size_t) ht * 8 + i] = a[i];
            }
            for (int ht = 0; ht < HT; ht++) {
                double2 a[8];
                for (int i = 0; i < 8; i++) a[i] = v[(size_t) ht * 8 + i];
                y_store1<PADV>(buf.data(), a, ht, t.w, p.ysh);
            }
        } else {
        for (int ht = 0; ht < HT; ht++) inv_pass<256>(buf.data(), tw2, ht);
        {
            std::vector<double2> v((size_t) HT * 16);
            for (int ht = 0; ht < HT; ht++) {
                double2 a[16];
                inv3_load(buf.data(), tw2, twf, ht, a);
                for (int i = 0; i < 16; i++) v[(size_t) ht * 16 + i] = a[i];
            }
            for (int ht = 0; ht < HT; ht++) {
                double2 a[16];
                for (int i = 0; i < 16; i++) a[i] = v[(size_t) ht * 16 + i];
                y_store<PADV>(buf.data(), a, ht, t.w, p.ysh);
            }
        }
        }
        if (s_i[0] > 0 && E.tc) {
            if constexpr (IR == 8) interp_tc<PADV>(p, dst, t, reinterpret_cast<const double*>(buf.data()), sbank.data(), s_goff.data(), s_i, s_o);
        } else if (s_i[0] > 0) {
            const double* yb = reinterpret_cast<const double*>(buf.data());
            const int n_tasks = TaskGeom<IR, GLOG>::n_tasks(p, s_i[1]);
            for (int task = 0; task < n_tasks; task++)
                for (int lane = 0; lane < 32; lane++) {
                    TaskGeom<IR, GLOG> g;
                    g.set(p, s_goff.data(), task, lane);
                    int yo[IQ2];
                    interp_windows<IR, GLOG>(p, g, s_i, yo);
                    double acc[IR][IQ2];
                    interp_acc<IR, PADV>(yb, sbank.data() + (size_t) g.grp * esz, yo, p.smaxp, p.ysh, acc);
                    interp_store_direct<IR, GLOG>(p, dst, t.ch, g, s_i, s_o, acc);
                }
        }
    }
}

template <int IR, bool PADV>
void run_glog(const FusedParams& p, const SrcView& src, const DstView& dst, const Emul& E)
{
    if (p.glog == 2) run_units<IR, PADV, 2>(p, src, dst, E);
    else if (p.glog == 1) run_units<IR, PADV, 1>(p, src, dst, E);
    else run_units<IR, PADV, 0>(p, src, dst, E);
}

} // namespace

extern "C" {

// A "2x BlockConvolver -> whole-stepping interpolator" resampler for ONE channel; returns NULL when the rate
// pair does not plan to that chain.
void* f2semul_create(double src, double dst, int max_in_len, double tb, double atten, int glog_force)
{
    Emul* E = new Emul;
    if (!E->plan.build(src, dst, max_in_len, tb, atten, 0, 0, 0) || E->plan.stages.size() != 2 ||
        E->plan.stages[1].kind != ST_FRAC_WHOLE) {
        delete E;
        return nullptr;
    }
    E->fg = fused_geometry(E->plan.stages[0], E->plan.stages[1]);
    if (!E->fg.ok) {
        delete E;
        return nullptr;
    }
    E->sched.init(&E->plan);
    E->tc = glog_force == 8 || E->fg.up == 1;
    E->B = build_group_bank(E->plan.stages[1], E->tc ? 8 : choose_group_ir(E->plan.stages[1]), E->tc);
    build_spectrum(E->plan.stages[0], 12, E->spec, E->tw, nullptr);
    E->tw_tab = build_tw_tab(E->tw);
    E->c_tab = build_c_tab(E->spec, E->tw, E->fg.up);
    if (E->fg.up == 2) E->cs_tab = build_cs_tab(E->plan.stages[0], E->tw);
    E->ring.assign((size_t) 1 << 22, 0.0);
    E->ring_mask = ((long long) 1 << 22) - 1;
    E->glog_force = E->tc ? -1 : glog_force;
    return E;
}

void f2semul_destroy(void* h) { delete (Emul*) h; }

// One process() call: l input samples at x (any alignment), up to out_cap outputs; returns the count.
int f2semul_process(void* h, const double* x, int l, double* out, int out_cap)
{
    Emul& E = *(Emul*) h;
    const int n_out = E.sched.advance(l, E.calls);
    if (n_out > out_cap) return -1;
    const StageCall& c = E.calls[0];
    const StageCall& fc = E.calls[1];
    const StageDesc& f = E.plan.stages[1];
    if (n_out > 0) {
        FusedParams p;
        memset(&p, 0, sizeof p);
        fused_whole_fields(p, f, fc.e0, fc.e1);
        fused2_tiles(p, E.fg, (int) (c.n0 & 1));
        p.yl = E.fg.yl;
        p.lg = E.fg.lg;
        p.ysh = E.fg.ysh;
        p.spec = E.spec.data();
        p.tw = E.tw.data();
        p.c_tab = E.c_tab.data();
        p.cs_tab = E.cs_tab.data();
        p.up = E.fg.up;
        p.ylen = E.fg.up * 4096;
        p.gbank = E.B.gb.data();
        p.goff = E.B.go.data();
        p.smaxp = E.B.smaxp;
        p.ir = E.B.ir;
        p.gbank_smem_len = E.B.n_groups * E.B.smaxp * E.B.ir;
        p.n_ch = 1;
        p.mbu = fused2_choose_mbu(p.span, f.in_step, f.out_step);
        p.glog = E.tc ? 0 : E.glog_force >= 0 ? E.glog_force : fused2_choose_glog(p.span, f.in_step, f.out_step, p.ir);
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
        dst.base = fc.e0;
        const bool pad = p.ysh != 31;
        if (p.ir == 10) {
            if (pad) run_glog<10, true>(p, src, dst, E);
            else run_glog<10, false>(p, src, dst, E);
        } else {
            if (pad) run_glog<8, true>(p, src, dst, E);
            else run_glog<8, false>(p, src, dst, E);
        }
    }
    for (int i = 0; i < l; i++) E.ring[(size_t) ((c.n0 + i) & E.ring_mask)] = x[i];
    return n_out;
}

// Every 2x BlockConvolver stage of the plan whose polyphase branches fit a 4096-point tile: all 4096 bins of G rebuilt
// from build_cs_tab() with the kernel's arithmetic (phi(kappa_t) = rot32<t>(phi_g), cs_bin_lo / cs_bin_hi) against
// build_spectrum()'s slot-ordered table.  out[0] = worst |difference| in units of ulp(max |G|) over those stages.
// Returns the number of stages compared, -1 when the plan is refused.
int f2semul_table_err(double src, double dst, int max_in, double tb, double atten, int extfft, double* out)
{
    Plan P;
    if (!P.build(src, dst, max_in, tb, atten, 0, extfft, 0)) return -1;
    int n = 0;
    out[0] = 0.0;
    for (const StageDesc& s : P.stages) {
        if (s.kind != ST_BLOCKCONV || s.up != 2 || s.down != 1 || s.block_exact || (s.lp.half_len + 1) / 2 >= FN) continue;
        std::vector<double2> spec, tw;
        build_spectrum(s, 12, spec, tw, nullptr);
        const std::vector<double2> cs = build_cs_tab(s, tw);
        double gmax = 0.0;
        for (const double2& v : spec) gmax = std::max(gmax, std::max(std::fabs(v.x), std::fabs(v.y)));
        const double ulp = gmax * 0x1p-52;
        for (int g = 0; g < HT; g++) {
            const int k0 = (g >> 4) + 16 * (g & 15), i2 = cs_second(g);
            const double2 phg = cs[(size_t) CS_PAIRS + HT + g];
            for (int t = 0; t < 8; t++) {
                double2 ph;
                switch (t) {
                case 0: ph = rot32<0>(phg); break;
                case 1: ph = rot32<1>(phg); break;
                case 2: ph = rot32<2>(phg); break;
                case 3: ph = rot32<3>(phg); break;
                case 4: ph = rot32<4>(phg); break;
                case 5: ph = rot32<5>(phg); break;
                case 6: ph = rot32<6>(phg); break;
                default: ph = rot32<7>(phg); break;
                }
                const int k = k0 + 256 * t;
                const double2 lo = cs_bin_lo(cs[(size_t) (g + 256 * t)], ph), hi = cs_bin_hi(cs[(size_t) (i2 - 256 * t)], ph);
                const double2 rl = spec[(size_t) slot_of<FM>(k)], rh = spec[(size_t) slot_of<FM>(k + FN)];
                const double e = std::max(std::max(std::fabs(lo.x - rl.x), std::fabs(lo.y - rl.y)),
                                          std::max(std::fabs(hi.x - rh.x), std::fabs(hi.y - rh.y)));
                out[0] = std::max(out[0], e / ulp);
            }
        }
        n++;
    }
    return n;
}

// Entries of a thread's two table reads at t = 0 (the kernel's indices; t moves them by +-256 t).
void f2semul_entries(int* first, int* second)
{
    for (int g = 0; g < HT; g++) {
        first[g] = g;
        second[g] = cs_second(g);
    }
}

// The per-plan shared-memory decision of batch_create for every stage that runs on k_up2_frac2 with UP = 2: 4 ints per
// stage -- kind (1: fused with the interpolator that follows, 2: the BlockConvolver alone), the largest bank it may hold
// (doubles), whether the symmetric spectrum table is kept in shared memory, and the dynamic shared memory of the launch
// with the table and without staging (bytes).  Returns the number of such stages, -1 when the plan is refused.
int f2semul_fit(double src, double dst, int max_in, double tb, double atten, int extfft, int* out, int cap)
{
    Plan P;
    if (!P.build(src, dst, max_in, tb, atten, 0, extfft, 0)) return -1;
    int n = 0;
    for (size_t i = 0; i < P.stages.size(); i++) {
        const StageDesc& s = P.stages[i];
        if (s.kind != ST_BLOCKCONV) continue;
        int kind = 0, bank = 0;
        const FusedGeom fg = i + 1 < P.stages.size() ? fused_geometry(s, P.stages[i + 1]) : FusedGeom();
        if (fg.ok && fg.up == 2) {
            kind = 1;
            bank = fused2_bank_doubles_max(P.stages[i + 1]);
        } else {
            const BcTile bt = blockconv_tile(s);
            if (!bt.large && s.up == 2 && s.down == 1 && !s.block_exact && 2 * (4096 - 2 * bt.lg) >= 2048) kind = 2;
        }
        if (kind == 0) continue;
        if (n < cap) {
            int* o = out + 4 * n;
            o[0] = kind;
            o[1] = bank;
            o[2] = fused2_cs_fits(bank) ? 1 : 0;
            o[3] = fused2_smem_bytes(bank, true, false);
        }
        n++;
    }
    return n;
}

} // extern "C"

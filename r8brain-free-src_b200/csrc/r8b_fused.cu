// r8b_fused.cu -- fused "2x BlockConvolver -> FracInterpolator" kernel: the 2x-rate stream never
// touches HBM.  This is the whole CDSPResampler::process() chain of BASELINE configs 1/2/3/5
// (CDSPResampler.h:218-333 case "upsampling or fractional downsampling down to 2X",
// CDSPBlockConvolver.h:252-354 + CDSPFracInterpolator.h:861-1179) in ONE launch per call.
//
// One CTA (512 threads) = one channel x one PAIR of consecutive tiles (a,b):
//   A. gather x_a + i*x_b straight from global into registers, first DIF pass   (threads 0..255)
//   B. DIF passes 2,3                                                             (threads 0..255)
//   C. per frequency pair (k, M-k): split the packed spectrum, multiply by G, write Y_a -> bufB and
//      Y_b -> bufA in place                                                      (all threads)
//   D. both inverse transforms side by side (thread>>8 selects the buffer); the last pass stores
//      the 2x-rate samples y[2m], y[2m+1] as plain doubles in an interpolation-friendly layout
//   E. fractional-delay interpolation from shared memory, results written to global:
//        whole stepping : register tile of R=8 output phases x Q=3 stepping cycles per lane;
//                         lanes = different cycles (distinct y addresses, conflict-free by
//                         construction of the layout), phase = warp-uniform (bank rows broadcast)
//        order-2 bank   : one output per thread, exact reference timing arithmetic
// Tiles own disjoint ranges of the 2x-rate position p; each tile's valid y range overlaps its
// neighbours by one interpolation window so no state is exchanged between CTAs.
#include "r8b_kernels.h"

#include <climits>

#include "r8b_fused_common.cuh"
#include "r8b_poly.cuh"
#include "r8b_interp.cuh"

namespace r8bgpu {

namespace {

constexpr int FNT = 512;            // threads per CTA
// interpolation register tile: IR output phases per lane (8 or 10, chosen per plan so that the
// number of phase groups divides evenly over the 16 warps) x IQ stepping cycles per lane
constexpr int IQ = 3;               // ... x stepping cycles per lane

// forward pass 1 fused with the gather from global memory (radix 16, NCUR = M, D = 256)
__device__ __forceinline__ void gather_loads(double2 (&v)[16], const SrcView& src, int ch, long long wa, long long wb,
                                             bool has_b, int r)
{
    // Interior tiles lie completely inside the caller's block: plain coalesced loads.  Only the
    // first tiles of a call reach back into the history ring (or ahead of the available input).
    const bool fast = wa >= src.cur_base && wb + FM <= src.avail && has_b;
    if (fast) {
        const double* __restrict__ pa = src.cur + (long long) ch * src.cur_stride + (wa - src.cur_base) + r;
        const double* __restrict__ pb = pa + (wb - wa);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            v[j].x = __ldg(pa + 256 * j);
            v[j].y = __ldg(pb + 256 * j);
        }
    } else {
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int n = r + 256 * j;
            v[j].x = src_read_f(src, ch, wa + n);
            v[j].y = has_b ? src_read_f(src, ch, wb + n) : 0.0;
        }
    }
}

__device__ __forceinline__ void fwd_pass1_regs(double2 (&v)[16], double2* __restrict__ s, const double2* __restrict__ twc,
                                               const double2* __restrict__ twf, int r)
{
    Network<16, +1>::run(v);
    s[fft_pad(r)] = v[0];
    twiddles16([&](int q) { return tw_pair(twc, twf, r, q); },
               [&](int q, double2 w) { s[fft_pad(r + q * 256)] = cmul<+1>(v[bitrev<16>(q)], w); });
}

// Pair-level bookkeeping for the whole-stepping interpolation, done by ONE thread at kernel start (it
// depends only on the launch parameters, so its 64-bit divisions hide behind the input gather).  Everything the
// per-task code needs afterwards is 32-bit and relative to the pair.  With delta = e0 mod 8 (out_step % 8 == 0)
// the phase groups are shifted so that every 8-phase row starts on a 64-byte boundary of the caller's buffer.
__device__ __forceinline__ void interp_prepare(const FusedParams& p, const DstView& dst, int ch, long long ya0,
                                               long long yb0, long long bsel, long long A0, long long B1, int* s_i,
                                               double** s_op)
{
    long long ja = (A0 * p.out_step + p.in_step - 1) / p.in_step;
    long long jb = (B1 * p.out_step + p.in_step - 1) / p.in_step;
    if (ja < p.e0) ja = p.e0;
    if (jb > p.e1) jb = p.e1;
    const long long ad = ja - p.delta, bd = jb - 1 - p.delta; // floor divisions (ad may be slightly negative)
    const long long c_first = ad >= 0 ? ad / p.out_step : -1, c_last = bd >= 0 ? bd / p.out_step : -1;
    s_i[0] = jb > ja ? (int) (jb - ja) : 0;                               // outputs of this pair
    s_i[1] = (int) (c_last - c_first);                                    // last (shifted) cycle, relative
    s_i[2] = (int) (c_first * p.out_step - ja);                           // output index of (cycle 0, phase 0) rel. to ja
    s_i[3] = (int) (c_first * p.in_step - p.fll - ya0);                   // y window start of (cycle 0, offset 0) in tile a
    s_i[4] = (bsel == LLONG_MAX || bsel - ya0 > 0x3fffffff) ? 0x3fffffff : (int) (bsel - ya0);
    s_i[5] = (int) (yb0 - ya0);
    *s_op = dst.ptr + (long long) ch * dst.stride + ((ja - dst.base) & dst.mask);
}

// Whole-stepping interpolation of one tile pair out of shared memory.  Task = (group of IR
// consecutive output phases) x (chunk of 32*IQ stepping cycles); lane = cycle, so the y reads of
// a warp are in_step doubles apart (conflict-free: odd stride, or made odd by the PAD layout) and the
// bank reads are warp-uniform broadcasts.  The tap loop is split into a predicated ramp-up, a
// branch-free middle where all IR phases are active, and a predicated ramp-down.
template <int IR, bool PAD, bool BANK_SMEM>
__device__ __forceinline__ void interp_whole(const FusedParams& p, const DstView& dst, int ch,
                                             const double* __restrict__ smd, int off_a, int off_b,
                                             long long ya0, long long yb0, long long bsel, long long A0,
                                             long long B1, const double* __restrict__ bank, double* stage,
                                             const int* __restrict__ s_i, double* const* s_op,
                                             const int* __restrict__ s_goff, int tid)
{
    constexpr int YMAX = 2 * FM;
    (void) ya0; (void) yb0; (void) bsel; (void) A0; (void) B1;
    double* const s_o = *s_op;
    const int n_j = s_i[0];
    if (n_j <= 0) return;
    const int c_cnt = s_i[1], jshift = s_i[2], wbase = s_i[3], bsel_r = s_i[4], yb_d = s_i[5];
    const int warp = tid >> 5, lane = tid & 31;
    const int n_groups = (p.out_step + IR - 1) / IR;
    const int n_chunks = (c_cnt + 32 * IQ) / (32 * IQ);
    const int n_tasks = n_groups * n_chunks;
    const int smaxp = p.smaxp;
    for (int task = warp; task < n_tasks; task += FNT / 32) {
        const int grp = task % n_groups, chunk = task / n_groups;
        const int r0 = p.delta + grp * IR; // first phase of the group (phases past out_step wrap into the next cycle)
        const int o0 = s_goff[grp];
        // group bank: [smaxp][IR] coefficients, phase r's filter pre-shifted by its window offset and
        // zero-padded, so the tap loop below has no predicates and one base address
        const double* __restrict__ gb = bank + (BANK_SMEM ? grp : r0) * smaxp * IR;
        int yo[IQ];
#pragma unroll
        for (int q = 0; q < IQ; q++) {
            int c = chunk * (32 * IQ) + q * 32 + lane;
            if (c > c_cnt) c = c_cnt;
            const int ws = c * p.in_step + o0 + wbase; // relative to tile a's first double
            const bool use_b = ws >= bsel_r;
            int li = use_b ? ws - yb_d : ws;
            if (li < 0) li = 0; // edge-cycle phases this pair does not own: never stored
            if (li > YMAX - smaxp) li = YMAX - smaxp;
            yo[q] = li + (PAD ? 0 : (use_b ? off_b : off_a));
            if (PAD) yo[q] |= use_b ? 0 : (1 << 30); // buffer select kept in bit 30 (layout applied per load)
        }
        auto yload = [&](int q, int s) -> double {
            if (!PAD) return smd[yo[q] + s];
            const int i = (yo[q] & ~(1 << 30)) + s;
            return smd[((yo[q] >> 30) ? off_a : off_b) + i + (i >> p.ysh)];
        };
        double acc[IR][IQ];
#pragma unroll
        for (int r = 0; r < IR; r++)
#pragma unroll
            for (int q = 0; q < IQ; q++) acc[r][q] = 0.0;
#ifdef R8BGPU_EXPERIMENTS
        const int s_end = (p.debug & 2) ? 0 : smaxp; // profiling experiment: skip the tap loop
#else
        const int s_end = smaxp;
#endif
#pragma unroll 4
        for (int s = 0; s < s_end; s++) { // smaxp is a multiple of 4
            double yv[IQ];
#pragma unroll
            for (int q = 0; q < IQ; q++) yv[q] = yload(q, s);
#pragma unroll
            for (int r = 0; r < IR; r += 2) {
                const double2 b = *reinterpret_cast<const double2*>(gb + s * IR + r); // warp-uniform
#pragma unroll
                for (int q = 0; q < IQ; q++) {
                    acc[r][q] = fma(b.x, yv[q], acc[r][q]);
                    acc[r + 1][q] = fma(b.y, yv[q], acc[r + 1][q]);
                }
            }
        }
        // Each lane owns IR consecutive outputs of ITS cycle (one 64-byte row; rows of neighbouring lanes
        // are out_step samples apart).  Storing straight from registers makes every STG.128 touch 32
        // different rows (lg_throttle was ~20 % of the kernel).  With a per-warp staging area the warp
        // transposes 4x4 blocks of 16-byte chunks so that 4 adjacent lanes write one whole row: 8 rows x
        // 64 B per instruction.  Row r lives at prow(r)*64 B with its chunks XOR-swizzled -- both the
        // row-wise writes and the transposed reads are bank-conflict free.
        const bool linear = (dst.mask == -1);
        double* const obase = s_o;
#ifdef R8BGPU_EXPERIMENTS
        if (p.debug & 1) { // profiling experiment: skip the stores
            if (acc[0][0] == 1.2345e300) obase[0] = acc[1][1]; // keep the loop alive
            continue;
        }
#endif
        if (linear && stage != nullptr && IR == 8) {
            double* const stg = stage + warp * 256;
            const int wrow = (lane ^ ((lane >> 2) & 1)) * 8, wsw = (lane >> 1) & 3;
#pragma unroll
            for (int q = 0; q < IQ; q++) {
                const int cb = chunk * (32 * IQ) + q * 32; // cycle of lane 0
                if (cb > c_cnt) break;
#pragma unroll
                for (int i = 0; i < 4; i++)
                    *reinterpret_cast<double2*>(stg + wrow + 2 * (i ^ wsw)) = make_double2(acc[2 * i][q], acc[2 * i + 1][q]);
                __syncwarp();
                const int ci = lane & 3;
#pragma unroll
                for (int t = 0; t < 4; t++) {
                    const int R = (lane & ~3) + t;
                    const double2 v = *reinterpret_cast<const double2*>(
                        stg + (R ^ ((R >> 2) & 1)) * 8 + 2 * (ci ^ ((R >> 1) & 3)));
                    const int c = cb + R;
                    const int j = c * p.out_step + r0 + jshift + 2 * ci; // first of this lane's two outputs
                    if (c > c_cnt) continue;
                    double* o = obase + j;
                    const bool in0 = (p.wrap || r0 + 2 * ci < p.out_step) && j >= 0 && j < n_j;
                    const bool in1 = (p.wrap || r0 + 2 * ci + 1 < p.out_step) && j + 1 >= 0 && j + 1 < n_j;
                    if (in0 && in1 && ((reinterpret_cast<unsigned long long>(o) & 15) == 0)) {
                        *reinterpret_cast<double2*>(o) = v; // (__stcs / __stwt measured within noise of the default)
                    } else {
                        if (in0) o[0] = v.x;
                        if (in1) o[1] = v.y;
                    }
                }
                __syncwarp();
            }
            continue;
        }
#pragma unroll
        for (int q = 0; q < IQ; q++) {
            const int c = chunk * (32 * IQ) + q * 32 + lane;
            if (c > c_cnt) continue;
            const int j0 = c * p.out_step + r0 + jshift; // relative to the pair's first output
            const bool full = (p.wrap || r0 + IR <= p.out_step) && j0 >= 0 && j0 + IR <= n_j;
            if (linear) {
                double* o = obase + j0;
                if (full) {
                    if ((reinterpret_cast<unsigned long long>(o) & 15) == 0) {
#pragma unroll
                        for (int r = 0; r < IR; r += 2)
                            *reinterpret_cast<double2*>(o + r) = make_double2(acc[r][q], acc[r + 1][q]);
                    } else { // 8-byte aligned start: scalar head and tail, aligned pairs in between
                        o[0] = acc[0][q];
#pragma unroll
                        for (int r = 1; r + 1 < IR; r += 2)
                            *reinterpret_cast<double2*>(o + r) = make_double2(acc[r][q], acc[r + 1][q]);
                        o[IR - 1] = acc[IR - 1][q];
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < IR; r++)
                        if ((p.wrap || r0 + r < p.out_step) && j0 + r >= 0 && j0 + r < n_j) o[r] = acc[r][q];
                }
            } else {
                // ring destination (another stage follows)
#pragma unroll
                for (int r = 0; r < IR; r++)
                    if ((p.wrap || r0 + r < p.out_step) && j0 + r >= 0 && j0 + r < n_j)
                        dst.ptr[(long long) ch * dst.stride + (((obase - (dst.ptr + (long long) ch * dst.stride)) + (long long) j0 + r) & dst.mask)] = acc[r][q];
            }
        }
    }
}

} // namespace

// MODE 0: whole stepping, MODE 1: order-2 polynomial bank.
// ---- order-2 bank (non-whole stepping) helpers ------------------------------------------------
// One thread, at kernel start: the pair's output range [ka, kb) -> s_j, rows of chunk 0 -> s_i[0..1].
__device__ __forceinline__ void poly_prepare(const FusedParams& p, long long A0, long long B1, int* s_j, int* s_i)
{
    const long long nk = p.e1 - p.e0;
    const long long ka = poly_first_k(p, A0, nk), kb = poly_first_k(p, B1, nk);
    s_j[0] = (int) ka;
    s_j[1] = (int) kb;
    int r_lo, n_st;
    poly_rows_for(p, ka, poly_chunk_start(ka, kb, 1, p.poly_chunks), r_lo, n_st);
    s_i[0] = r_lo;
    s_i[1] = n_st;
}

// Copy rows (r_lo + s) mod fracs, s < n_st, into shared memory with threads t0, t0 + nthr, ...
__device__ __forceinline__ void poly_stage_rows(const FusedParams& p, double* sbank, int r_lo, int n_st, int t0, int nthr)
{
    const int rl2 = (3 * p.flen) >> 1; // double2 per row (flen is even whenever rows are staged)
    double2* sb2 = reinterpret_cast<double2*>(sbank);
    const double2* gb2 = reinterpret_cast<const double2*>(p.bank);
    for (int i = t0; i < n_st * rl2; i += nthr) {
        const int sl = i / rl2;
        int row = r_lo + sl;
        if (row >= p.fracs) row -= p.fracs;
        sb2[sl * (p.poly_row_stride >> 1) + (i - sl * rl2)] = __ldg(gb2 + (long long) row * rl2 + (i - sl * rl2));
    }
}

// ---- order-2 bank: the output loop ------------------------------------------------------------
struct PolyCtx {
    const double* smd;    // dynamic shared memory as doubles: tile b's y at 0, tile a's y at 2*FPL
    const double* sbank;  // staged rows: slot s holds row (r_lo + s) mod fracs
    int r_lo, n_st;
    long long ya0, yb0;   // absolute 2x index of y element 0 of tile a / tile b
    long long bsel;       // windows starting at or after this position use tile b
    int ch;
    int* queue;           // outputs deferred to the one-output-per-lane pass (POLY_QUEUE entries)
    int* q_count;
};

template <bool PADV>
__device__ __forceinline__ double poly_single(const FusedParams& p, const PolyCtx& cx, const PolyOut& o)
{
    const double* yb = cx.smd + (o.use_b ? 0 : 2 * FPL);
    const int yi = o.yi, ysh = p.ysh;
    auto y = [=](int i) { return PADV ? yb[ylay(yi + i, ysh)] : yb[yi + i]; };
    const int rowlen = 3 * p.flen;
    const int slot = poly_slot(p, cx.r_lo, o.fti);
    if (slot < cx.n_st && o.fti < p.fracs)
        return poly_row_dot<true>(cx.sbank + slot * p.poly_row_stride, p.flen, o.x, o.x2, y);
    return poly_row_dot<false>(p.bank + (long long) o.fti * rowlen, p.flen, o.x, o.x2, y);
}

// Outputs [k_lo, k_hi) of one chunk.  N > 0: threads take four consecutive outputs; when these share a staged
// bank row and their windows start exactly N samples apart (the steady state of a slowly drifting ratio
// ~ N) the coefficient loads are shared (poly_block4), otherwise each output goes the single-output way.
// N == 0: one output per thread.
template <int N, bool PADV>
__device__ __forceinline__ void poly_outputs(const FusedParams& p, const DstView& dst, const PolyCtx& cx, int k_lo, int k_hi,
                                             int tid)
{
    if (N == 0) {
        for (int k = k_lo + tid; k < k_hi; k += FNT) {
            const PolyOut o = poly_output(p, cx.ya0, cx.yb0, cx.bsel, k);
            if (!o.ok) continue;
            dst_write_f(dst, cx.ch, p.e0 + k, poly_single<PADV>(p, cx, o));
        }
        return;
    }
    // Groups that do not qualify (the bank row changes inside the group, a tile boundary, the last few outputs)
    // are not computed in place -- a warp would serialise its few slow lanes behind the fast ones on every
    // pass -- but queued in shared memory and computed afterwards one output per lane, all lanes busy.
    constexpr int NN = N > 0 ? N : 1;
#ifdef R8BGPU_PHASE_TIMERS
    long long tq0 = clock64();
#endif
    for (int k = k_lo + 4 * tid; k < k_hi; k += 4 * FNT) {
        PolyOut o[4];
        const int nv = min(4, k_hi - k);
#pragma unroll
        for (int r = 0; r < 4; r++)
            if (r < nv) o[r] = poly_output(p, cx.ya0, cx.yb0, cx.bsel, k + r);
        int slot;
        if (poly_fast_group<NN>(p, o, nv, cx.r_lo, cx.n_st, slot)) {
            const double* yb = cx.smd + (o[0].use_b ? 0 : 2 * FPL);
            const int yi = o[0].yi, ysh = p.ysh;
            auto y = [=](int j) { return PADV ? yb[ylay(yi + j, ysh)] : yb[yi + j]; };
            const double xs[4] = {o[0].x, o[1].x, o[2].x, o[3].x};
            const double x2s[4] = {o[0].x2, o[1].x2, o[2].x2, o[3].x2};
            double acc[4];
            poly_block4<NN>(cx.sbank + slot * p.poly_row_stride, p.flen, xs, x2s, y, acc);
#pragma unroll
            for (int r = 0; r < 4; r++) dst_write_f(dst, cx.ch, p.e0 + k + r, acc[r]);
        } else {
            const int at = atomicAdd(cx.q_count, nv);
#pragma unroll
            for (int r = 0; r < 4; r++) {
                if (r >= nv) continue;
                if (at + r < POLY_QUEUE) cx.queue[at + r] = k + r;
                else if (o[r].ok) dst_write_f(dst, cx.ch, p.e0 + k + r, poly_single<PADV>(p, cx, o[r])); // queue full
            }
        }
    }
    __syncthreads();
#ifdef R8BGPU_PHASE_TIMERS
    if (p.prof != nullptr && tid == 0) {
        const long long t = clock64();
        atomicAdd(&p.prof[8], (unsigned long long) (t - tq0));
        tq0 = t;
    }
#endif
    const int nq = min(*cx.q_count, POLY_QUEUE);
    for (int i = tid; i < nq; i += FNT) {
        const int k = cx.queue[i];
        const PolyOut o = poly_output(p, cx.ya0, cx.yb0, cx.bsel, k);
        if (o.ok) dst_write_f(dst, cx.ch, p.e0 + k, poly_single<PADV>(p, cx, o));
    }
#ifdef R8BGPU_PHASE_TIMERS
    if (p.prof != nullptr) {
        __syncthreads();
        if (tid == 0) atomicAdd(&p.prof[9], (unsigned long long) (clock64() - tq0));
    }
#endif
}

template <int MODE, int IRV, bool PADV, bool BANKV>
__global__ void __launch_bounds__(FNT, 1) k_up2_frac(FusedParams p, SrcView src, DstView dst)
{
    extern __shared__ double2 smem[];
    double2* bufA = smem;              // forward spectrum Z, later Y_b / y_b
    double2* bufB = smem + FPL;        // Y_a / y_a
    double2* tw2 = smem + 2 * FPL;     // tw2t[q*16+r] = W_256^(r q)
    double2* twc = tw2;                // (same table: coarse factor of the NCUR = M twiddles)
    double2* twf = tw2 + 256;          // tw1t[q*16+r] = W_M^(r q)
    double* sbank = reinterpret_cast<double*>(twf + 256); // whole-step bank (if it fits)
    __shared__ int s_j[2];
    __shared__ int s_q;
    __shared__ int s_i[8];
    __shared__ double* s_o;
    __shared__ int s_goff[192];

    const int tid = threadIdx.x;
    const int n_pairs = (p.n_tiles + 1) >> 1;
    const int ch = blockIdx.x / n_pairs;
    const int pair = blockIdx.x - ch * n_pairs;
    const int ta = 2 * pair;
    const bool has_b = (ta + 1) < p.n_tiles;
    // owned 2x-rate position ranges [A0,A1) and [B0,B1)
    const long long A0 = p.p_lo + (long long) ta * p.span;
    long long A1 = A0 + p.span;
    if (A1 > p.p_hi) A1 = p.p_hi;
    const long long B0 = A1;
    long long B1 = has_b ? B0 + p.span : B0;
    if (B1 > p.p_hi) B1 = p.p_hi;
    // valid y of tile t starts at own_start - YL (even) = 2 * (first valid m); window starts lg earlier
    const long long wa = (A0 - p.yl) / 2 - p.lg;
    const long long wb = (B0 - p.yl) / 2 - p.lg;

    // the input gather goes first (longest latency), the table loads ride behind it
    double2 gv[16];
    if (tid < 256) gather_loads(gv, src, ch, wa, wb, has_b, tid);
    // tables into shared memory
    {
        const int i = tid & 255, q = i >> 4, r = i & 15;
        if (tid < 256) tw2[i] = __ldg(&p.tw[(r * q) * (FM / 256)]);
        else twf[i] = __ldg(&p.tw[r * q]);
    }
    if (MODE == 0) {
        const int n_groups = (p.out_step + IRV - 1) / IRV, esz = p.smaxp * IRV;
        if (BANKV) {
            // threads 256..511 are otherwise idle during the forward transform: they fetch the bank entries of
            // this call's phase groups (first phases delta, delta+8, ...) into consecutive slots
            for (int i = tid - 256; i >= 0 && i < n_groups * esz; i += 256) {
                const int g = i / esz;
                sbank[i] = __ldg(&p.gbank[(long long) (p.delta + g * IRV) * esz + (i - g * esz)]);
            }
        }
        if (tid >= 256 && tid - 256 < n_groups) s_goff[tid - 256] = __ldg(&p.goff[p.delta + (tid - 256) * IRV]);
        if (tid == 511) {
            const long long bsel0 = has_b ? B0 - p.yl : LLONG_MAX;
            interp_prepare(p, dst, ch, 2 * wa, 2 * wb, bsel0, A0, B1, s_i, &s_o);
        }
    } else if (tid == 511) {
        poly_prepare(p, A0, B1, s_j, s_i);
    }
    __syncthreads();
    // threads idle during the forward transform stage the bank rows of the pair's first chunk
    if (MODE == 1 && tid >= 256) poly_stage_rows(p, sbank, s_i[0], s_i[1], tid - 256, 256);

    // optional phase timing: build with R8BGPU_PHASE_TIMERS=1 (adds -DR8BGPU_PHASE_TIMERS) and run with
    // R8BGPU_PROFILE=1; thread 0 accumulates clock64() deltas per phase.  Compiled out by default: the live
    // 64-bit timestamp was being spilled around every barrier.
#ifdef R8BGPU_PHASE_TIMERS
    long long t_prev = p.prof ? clock64() : 0;
#define R8B_TICK(i)                                                                  \
    if (p.prof != nullptr && tid == 0) {                                             \
        const long long t_now = clock64();                                           \
        atomicAdd(&p.prof[i], (unsigned long long) (t_now - t_prev));                \
        t_prev = t_now;                                                              \
    }
#else
#define R8B_TICK(i)
#endif
    if (tid < 256) fwd_pass1_regs(gv, bufA, twc, twf, tid);
    __syncthreads();
    R8B_TICK(0)
    if (tid < 256) fwd_pass<256>(bufA, tw2, tid);
    __syncthreads();
    R8B_TICK(1)
    if (tid < 256) fwd_pass<16>(bufA, tw2, tid);
    __syncthreads();
    R8B_TICK(2)

    // C. frequency pairs.  Only slots whose frequency k <= M/2 start a pair; in slot order those are the
    //    slots with low digit q3 < 8 (k = q1 + 16 q2 + 256 q3), plus k = M/2 (slot 8).  Thread t handles
    //    slots 16*((t>>3) + 64u) + (t&7): runs of 8 consecutive double2 (conflict-free), no idle iterations,
    //    and every spectrum value is fetched exactly once per CTA.
    {
        constexpr int NC = FM / (2 * FNT);
        double2 g1[NC], g2[NC];
        int s1v[NC], s2v[NC];
#pragma unroll
        for (int u = 0; u < NC; u++) {
            const int s1 = 16 * ((tid >> 3) + 64 * u) + (tid & 7);
            const int k = freq_of<FM>(s1);
            const int s2 = slot_of<FM>((FM - k) & (FM - 1));
            s1v[u] = s1;
            s2v[u] = s2;
            if (p.c_tab != nullptr) { // thread-ordered copy of the two spectrum values: a warp's loads are 512 contiguous bytes
                g1[u] = __ldg(&p.c_tab[(2 * u) * FNT + tid]);
                g2[u] = __ldg(&p.c_tab[(2 * u + 1) * FNT + tid]);
            } else {
                g1[u] = __ldg(&p.spec[s1]);
                g2[u] = __ldg(&p.spec[s2]);
            }
        }
        auto do_pair = [&](int s1, int s2, double2 ga, double2 gb) {
            const double2 z1 = bufA[fft_pad(s1)];
            const double2 z2 = bufA[fft_pad(s2)];
            // X_a[k] = z1 + conj z2 (the 1/2 lives in G); X_a[M-k] = conj X_a[k]
            const double2 xa = make_double2(z1.x + z2.x, z1.y - z2.y);
            const double2 xb = make_double2(z1.y + z2.y, z2.x - z1.x); // -i (z1 - conj z2)
            bufB[fft_pad(s1)] = cmul<+1>(xa, ga);
            bufA[fft_pad(s1)] = cmul<+1>(xb, ga);
            if (s2 != s1) {
                bufB[fft_pad(s2)] = cmul<+1>(make_double2(xa.x, -xa.y), gb);
                bufA[fft_pad(s2)] = cmul<+1>(make_double2(xb.x, -xb.y), gb);
            }
        };
#pragma unroll
        for (int u = 0; u < NC; u++) do_pair(s1v[u], s2v[u], g1[u], g2[u]);
        if (tid == 0) { // k = M/2 pairs with itself
            const int sh = slot_of<FM>(FM / 2);
            do_pair(sh, sh, __ldg(&p.spec[sh]), __ldg(&p.spec[sh]));
        }
    }
    __syncthreads();
    R8B_TICK(3)

    // D. two inverse transforms side by side
    {
        double2* buf = (tid < 256) ? bufB : bufA;
        const int g = tid & 255;
        inv_pass<16>(buf, tw2, g);
        __syncthreads();
        R8B_TICK(4)
        inv_pass<256>(buf, tw2, g);
        __syncthreads();
        R8B_TICK(5)
        // last pass: NCUR = M, D = 256, twiddle W_M^(r q) conj; results leave in y layout
        double2 v[16];
        v[0] = buf[fft_pad(g)];
        twiddles16([&](int q) { return tw_pair(twc, twf, g, q); },
                   [&](int q, double2 w) { v[q] = cmul<-1>(buf[fft_pad(g + q * 256)], w); });
        Network<16, -1>::run(v);
        __syncthreads();
        double* yb = reinterpret_cast<double*>(buf);
        const long long w = (tid < 256) ? wa : wb;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int e = g + j * 256;           // local input-rate position
            double2 x = v[bitrev<16>(j)];
            const long long t0 = 2 * (w + e);    // absolute 2x-rate index of x.x
            if (t0 < 0) x = make_double2(0.0, 0.0); // the reference's interpolator starts from silence
            if (!PADV) {
                reinterpret_cast<double2*>(yb)[e] = x; // plain layout: one 128-bit store
            } else {
                yb[ylay(2 * e, p.ysh)] = x.x;
                yb[ylay(2 * e + 1, p.ysh)] = x.y;
            }
        }
    }
    __syncthreads();
    R8B_TICK(6)

    const long long ya0 = 2 * wa, yb0 = 2 * wb;   // absolute 2x index of local double 0
    const long long bsel = has_b ? B0 - p.yl : LLONG_MAX; // windows starting at or after this use tile b

    if (MODE == 0) {
        const double* smd = reinterpret_cast<const double*>(smem);
        const int off_a = 2 * FPL, off_b = 0; // tile a lives in bufB, tile b in bufA (in doubles)
        interp_whole<IRV, PADV, BANKV>(p, dst, ch, smd, off_a, off_b, ya0, yb0, bsel, A0, B1, BANKV ? sbank : p.gbank,
                                       p.stage_off > 0 ? reinterpret_cast<double*>(smem) + p.stage_off : nullptr, s_i, &s_o,
                                       s_goff, tid);
    } else {
        // order-2 bank: output k of this call (k >= 0) sits at (p_k, fpos_k); the pair owns k in [ka, kb)
        // (found by poly_prepare at kernel start)
        const int ka = s_j[0], kb = s_j[1];
        int r_lo = s_i[0], n_st = s_i[1];
        const double* smd1 = reinterpret_cast<const double*>(smem);
        for (int c = 0; c < p.poly_chunks; c++) {
            const int k_lo = (int) poly_chunk_start(ka, kb, c, p.poly_chunks);
            const int k_hi = (int) poly_chunk_start(ka, kb, c + 1, p.poly_chunks);
            __syncthreads(); // everyone is done with the previous chunk's rows and queue
            if (tid == 0) s_q = 0;
            if (c > 0) { // next run of rows: every thread derives the same (r_lo, n_st); all threads copy
                poly_rows_for(p, k_lo, k_hi, r_lo, n_st);
                poly_stage_rows(p, sbank, r_lo, n_st, tid, FNT);
            }
            __syncthreads();
            PolyCtx cx;
            cx.smd = smd1;
            cx.sbank = sbank;
            cx.r_lo = r_lo;
            cx.n_st = n_st;
            cx.ya0 = ya0;
            cx.yb0 = yb0;
            cx.bsel = bsel;
            cx.ch = ch;
            cx.queue = reinterpret_cast<int*>(sbank + (size_t) p.poly_rows_cap * p.poly_row_stride);
            cx.q_count = &s_q;
            if (p.poly_n == 2) poly_outputs<2, PADV>(p, dst, cx, k_lo, k_hi, tid);
            else if (p.poly_n == 1) poly_outputs<1, PADV>(p, dst, cx, k_lo, k_hi, tid);
            else if (p.poly_n == 3) poly_outputs<3, PADV>(p, dst, cx, k_lo, k_hi, tid);
            else poly_outputs<0, PADV>(p, dst, cx, k_lo, k_hi, tid);
        }
    }
#ifdef R8BGPU_PHASE_TIMERS
    if (p.prof != nullptr) {
        __syncthreads();
        R8B_TICK(7)
    }
#endif
#undef R8B_TICK
}

int fused_max_span(int lg, int yl, int yr) { return 2 * (FM - 2 * lg) - yl - yr; }
int fused_stage_doubles() { return (FNT / 32) * 256; }              // 32 rows x 8 doubles per warp
int fused_fixed_doubles() { return 2 * (2 * FPL + 256 + 256); }     // buffers + twiddle tables

template <int MODE, int IRV, bool PADV, bool BANKV>
static void launch_inst(const FusedParams& p, const SrcView& src, const DstView& dst, int n_ch, int smem, cudaStream_t st,
                        FusedVariant* v)
{
    ensure_dyn_smem<k_up2_frac<MODE, IRV, PADV, BANKV>>(224 * 1024);
    const int n_pairs = (p.n_tiles + 1) >> 1;
    k_up2_frac<MODE, IRV, PADV, BANKV><<<(unsigned) (n_pairs * n_ch), FNT, smem, st>>>(p, src, dst);
    if (v != nullptr) {
        *v = FusedVariant();
        v->kernel = 1;
        v->mode = MODE;
        v->ir = IRV;
        v->pad = PADV;
        v->bank = BANKV;
    }
}

void launch_up2_frac(const FusedParams& p, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st, FusedVariant* v)
{
    if (p.n_tiles <= 0 || n_ch <= 0) return;
    int smem = fused_smem_bytes((p.mode == 0 && p.bank_in_smem) ? p.gbank_smem_len : 0);
    if (p.mode == 0 && p.stage_off > 0) smem = (p.stage_off + fused_stage_doubles()) * (int) sizeof(double);
    if (p.mode != 0) {
        smem = fused_poly_smem_bytes(p.poly_dir, p.poly_rows_cap, p.poly_row_stride); // what plan_poly_call reports
        if (p.ysh != 31) launch_inst<1, 8, true, false>(p, src, dst, n_ch, smem, st, v);
        else launch_inst<1, 8, false, false>(p, src, dst, n_ch, smem, st, v);
        return;
    }
    const bool pad = p.ysh != 31, bs = p.bank_in_smem != 0;
    // one kernel per (phases per group, y layout, bank location): registers are allocated per variant
    if (p.ir == 10) {
        if (!pad && bs) launch_inst<0, 10, false, true>(p, src, dst, n_ch, smem, st, v);
        else if (!pad) launch_inst<0, 10, false, false>(p, src, dst, n_ch, smem, st, v);
        else if (bs) launch_inst<0, 10, true, true>(p, src, dst, n_ch, smem, st, v);
        else launch_inst<0, 10, true, false>(p, src, dst, n_ch, smem, st, v);
    } else {
        if (!pad && bs) launch_inst<0, 8, false, true>(p, src, dst, n_ch, smem, st, v);
        else if (!pad) launch_inst<0, 8, false, false>(p, src, dst, n_ch, smem, st, v);
        else if (bs) launch_inst<0, 8, true, true>(p, src, dst, n_ch, smem, st, v);
        else launch_inst<0, 8, true, false>(p, src, dst, n_ch, smem, st, v);
    }
}

} // namespace r8bgpu

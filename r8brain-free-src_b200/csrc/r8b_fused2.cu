// r8b_fused2.cu -- v2 of the fused "BlockConvolver -> FracInterpolator" kernel (CDSPResampler.h:218-333;
// CDSPBlockConvolver.h:252-354 + CDSPFracInterpolator.h:991-1060): the whole process() chain of BASELINE configs 1/2/3,
// the tail of the decimating chains (UP = 1), and the lone 2x BlockConvolver of chains that continue with half-band
// upsamplers (COPY), in ONE launch per call.
//
// v1 (r8b_fused.cu) gives an SM to one 512-thread CTA that walks a tile pair through seven block-wide phases.  v2 is a
// PERSISTENT CTA per SM made of two independent 256-thread pipelines ("halves"): each half owns one tile at a time and
// synchronises only with itself (named barriers, bar.sync id,256), so one half's transforms run under the other half's
// interpolation.  (An mbarrier token makes the halves take turns at the interpolation -- flags bit 0; set per call where
// phase C reads the filter spectrum from shared memory, r8b_capi.cu.)  Shared tables arrive once per CTA
// by bulk async copy (cp.async.bulk + mbarrier): the [q][r] twiddle tables and this call's phase-group bank.  A tile's
// 4096 input samples are one contiguous 32 KB run of the caller's block or of the previous stage's ring: they are
// prefetched into L2 a tile ahead (cp.async.bulk.prefetch.L2) and land in the tile buffer's upper half by one bulk copy
// issued as soon as the half's previous tile has left the buffer; no registers are spent on prefetch.  Tiles at the
// edges of a call (history ring across a wrap, not yet available input), misaligned rows and typed (int16 .. float32)
// caller blocks are gathered with plain loads.
//
// Per tile: real-input forward FFT (2048 complex points), spectrum split x filter spectrum fused into the first inverse
// pass (UP = 2) or as its own phase (UP = 1), inverse FFT, then the whole-step interpolation as 16x8x16 fp64 matrix
// products (mma.sync m16n8k16 = DMMA) out of shared memory.  The arithmetic lives in r8b_fused2_core.cuh, which also
// compiles for the host (tests/cpp/fused2_emul.cpp).
//
// Shared memory: 2 tile buffers (4096 + 16 padded double2 each) + twiddles 8 KB + the call's bank + (UP = 2, where it fits)
// the filter spectrum in its symmetric half-size form, 32 KB (+ per-warp store staging for the FMA interpolation variants
// only, where that fits too) + the call's tile table (24 bytes per tile index, in what is left).
#include "r8b_kernels.h"

#include <algorithm>
#include <cstdint>
#include <type_traits>

#include "r8b_fused2_core.cuh"
#include "r8b_poly.cuh"

namespace r8bgpu {

namespace {

using namespace f2;

constexpr int NT2 = 2 * HT;
constexpr int STAGE_UP = fft_pad(FN);  // double2 index where a bulk-copied input tile lands (upper half of the buffer)

// ---- PTX helpers: named barriers, mbarriers, bulk async copies ---------------------------------
__device__ __forceinline__ void bar_half(int h) { asm volatile("bar.sync %0, 256;" ::"r"(h + 1) : "memory"); }
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* b, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* b)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(b)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* b)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(b))
                 : "memory");
}
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Transposed stores (IR == 8, linear destination): the lane's 8 outputs of one cycle are a 64-byte row;
// rows of neighbouring lanes are out_step samples apart, so storing straight from registers would touch 32
// rows per instruction.  Through a 2 KB per-warp staging area the warp transposes 4x4 blocks of 16-byte
// chunks so that 4 adjacent lanes write one whole row: 8 rows x 64 B per instruction (rows of the two
// phase groups of a cycle are adjacent: 128 B runs).  Row R lives at prow(R)*64 B with its chunks
// XOR-swizzled -- both the row-wise writes and the transposed reads are bank-conflict free.
template <int GLOG>
__device__ __forceinline__ void interp_store_staged(const FusedParams& p, const int* __restrict__ s_i, double* s_o, double* stg,
                                                    int task, int lane, const double (&acc)[8][IQ2])
{
    using G = TaskGeom<8, GLOG>;
    const int n_j = s_i[0], c_cnt = s_i[1], jshift = s_i[2];
    const int n_groups = (p.out_step + 7) / 8;
    const int n_gt = (n_groups + G::GL - 1) / G::GL;
    const int gt = task % n_gt, chunk = task / n_gt;
    const int wrow = (lane ^ ((lane >> 2) & 1)) * 8, wsw = (lane >> 1) & 3;
#pragma unroll
    for (int q = 0; q < IQ2; q++) {
        const int cq = chunk * G::CYC + q * G::CL; // cycle of cycle-lane 0
        if (cq > c_cnt) break;
#pragma unroll
        for (int i = 0; i < 4; i++)
            *reinterpret_cast<double2*>(stg + wrow + 2 * (i ^ wsw)) = make_double2(acc[2 * i][q], acc[2 * i + 1][q]);
        __syncwarp();
        const int ci = lane & 3;
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const int R = (lane & ~3) + t;
            const double2 v = *reinterpret_cast<const double2*>(stg + (R ^ ((R >> 2) & 1)) * 8 + 2 * (ci ^ ((R >> 1) & 3)));
            const int c = cq + (R & (G::CL - 1));
            const int grp = gt * G::GL + (R >> (5 - GLOG));
            if (c > c_cnt || grp >= n_groups) continue;
            const int r0 = p.delta + grp * 8;
            const int j = c * p.out_step + r0 + jshift + 2 * ci; // first of this lane's two outputs
            double* o = s_o + j;
            const bool in0 = (p.wrap || r0 + 2 * ci < p.out_step) && j >= 0 && j < n_j;
            const bool in1 = (p.wrap || r0 + 2 * ci + 1 < p.out_step) && j + 1 >= 0 && j + 1 < n_j;
            if (in0 && in1 && ((reinterpret_cast<unsigned long long>(o) & 15) == 0)) {
                *reinterpret_cast<double2*>(o) = v;
            } else {
                if (in0) o[0] = v.x;
                if (in1) o[1] = v.y;
            }
        }
        __syncwarp();
    }
}

} // namespace

// D = A(8x4, row) * B(4x8, col) + D on the fp64 tensor path (SASS: DMMA.8x8x4; the order-2 bank path)
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// D = A(16xKW, row) * B(KWx8, col) + D, KW = 16, 8 or 4 (SASS: DMMA.16x8x16, .16x8x8, .16x8x4); fragments in
// r8b_fused2_core.cuh (mma_a_index, mma_b_index, mma_store)
template <int KW>
__device__ __forceinline__ void dmma16(double (&c)[4], const double (&a)[KW / 2], const double (&b)[KW / 4])
{
    if constexpr (KW == 16)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                     "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
                       "d"(b[2]), "d"(b[3]));
    else if constexpr (KW == 8)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    else
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(b[0]));
}

// flags: bit 0 = ping-pong token around the interpolation, bit 1 = bulk-copy input tiles
// TC: interpolation as 16x8x16 fp64 matrix products (IRV == 8; GLOG unused)
// UP: up-factor of the BlockConvolver (2: 4096-point complex inverse, 8192 stream samples per tile; 1: 2048-point inverse
// mirroring the real-input forward transform, 4096 samples per tile -- TC only)
// COPY: no interpolator follows -- phase E writes the tile's owned positions of the 2x-rate stream to the destination
// (the BlockConvolver 2/1 alone: chains that continue with half-band upsamplers, or end there); no bank is loaded.
// POLY: the interpolator is the order-2 bank (CDSPFracInterpolator::convolve2, CDSPFracInterpolator.h:1069-1179) of a
// ratio close to an integer N: eight consecutive outputs whose windows start N samples apart and whose bank rows are two
// neighbours {r, r+1} form a GEMM  D[j][n] = sum_i y[p_j + i] * B[i][n]  with B's columns = (c0, c1, c2) of the two rows;
// output j = D[j][c0] + x_j D[j][c1] + x_j^2 D[j][c2] of its own row.  Blocks that do not fit (a position slip, the row
// index wrapping) are computed one output per quad from the bank in global memory.
// CS (UP = 2): phase C reads the filter spectrum in its symmetric half-size form from shared memory (FusedParams::cs_tab),
// else the full table from global memory (cd_tab).  A template parameter: with both paths in one kernel the register
// allocation of the whole kernel gets worse (spills).
// LIN (TC only): the destination is linear fp64, so the tensor path's stores compile to that case alone (mma_store).
template <int IRV, bool PADV, int GLOG, bool TC, int UP = 2, bool COPY = false, bool POLY = false, bool CS = false, bool LIN = false>
__global__ void __launch_bounds__(NT2, 1) k_up2_frac2(const __grid_constant__ FusedParams p, const __grid_constant__ SrcView src,
                                                      const __grid_constant__ DstView dst)
{
    extern __shared__ __align__(128) double2 smem[];
    double2* const tw2 = smem + 2 * FPL2;         // tw2t[q*16+r] = W_256^(r q)
    double2* const twf = tw2 + 256;               // tw1t[q*16+r] = W_M^(r q)
    double* const sbank = reinterpret_cast<double*>(twf + 256);
    const int n_groups = (p.out_step + IRV - 1) / IRV, esz = p.smaxp * IRV;
    const int n_bank = (COPY || POLY) ? 0 : n_groups;
    static_assert(!CS || UP == 2, "the symmetric spectrum table is the 2x pair's");
    // phase C's spectrum pairs after the bank (where the plan has room for them; else they are read from cd_tab)
    double2* const scs = reinterpret_cast<double2*>(sbank + ((n_bank * esz + 1) & ~1));
    // the call's tile table (r8b_fused2_core.cuh, TileEntry), after everything else
    TileEntry* const tab = reinterpret_cast<TileEntry*>(reinterpret_cast<char*>(smem) + p.tab_off);
    __shared__ __align__(8) unsigned long long mb[5]; // 0: tables, 1-2: input tile of half h, 3-4: interpolation turn of half h
    __shared__ TileEntry s_te[2];                     // entry of half h's tile where the table has none (ti >= n_tab)
    __shared__ int s_goff[192];

    const int tid = threadIdx.x, h = tid >> 8, ht = tid & (HT - 1), lane = tid & 31, wh = ht >> 5;
    double2* const buf = smem + h * FPL2;
    const int n_units = p.n_tiles * p.n_ch;
    const bool pingpong = (p.flags & 1) != 0, tma_in = (p.flags & 2) != 0;

    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 5; i++) mbar_init(&mb[i], 1);
        fence_mbar_init();
    }
    if (!COPY && !POLY && tid < n_groups) s_goff[tid] = __ldg(&p.goff[p.delta + tid * IRV]);
    if (!COPY)
        for (int i = tid; i < p.n_tab; i += NT2) tab[i] = tile_entry(p, dst.base, i);
    __syncthreads();
    if (tid == 0) {
        // tables: one transaction barrier, 1 + n_groups (+ 1) bulk copies
        mbar_expect_tx(&mb[0], (uint32_t) (512 * sizeof(double2) + (size_t) n_bank * esz * sizeof(double) +
                                           (CS ? CS_PAIRS * sizeof(double2) : 0)));
        bulk_g2s(tw2, p.tw_tab, 512 * sizeof(double2), &mb[0]);
        if (CS) bulk_g2s(scs, p.cs_tab, CS_PAIRS * sizeof(double2), &mb[0]);
        for (int g = 0; g < n_bank; g++)
            bulk_g2s(sbank + g * esz, p.gbank + (long long) (p.delta + g * IRV) * esz, (uint32_t) (esz * sizeof(double)), &mb[0]);
        mbar_arrive(&mb[3]); // half 0 interpolates first
    }

    const int stride = 2 * (int) gridDim.x;
    int u = 2 * (int) blockIdx.x + h;
    uint32_t par_in = 0, par_turn = 0;
    Tile t;
    int path = -1;
    auto tile_src = [&](const Tile& tt) { return tile_run(src, tt); };
    if (u < n_units) {
        t = tile_of(p, u);
        path = tile_input_path(src, t);
        if (path == 2 && !tma_in) path = 1;
        if (path == 2 && ht == 0) {
            mbar_expect_tx(&mb[1 + h], FM * sizeof(double));
            bulk_g2s(buf + STAGE_UP, tile_src(t), FM * sizeof(double), &mb[1 + h]);
        }
    }
    mbar_wait(&mb[0], 0); // twiddles, bank and spectrum pairs have landed

    // optional phase timing: build with R8BGPU_PHASE_TIMERS=1 (adds -DR8BGPU_PHASE_TIMERS) and run with R8BGPU_PROFILE=1;
    // thread 0 of each half accumulates clock64() deltas per phase of its tiles into p.prof:
    //   0 A_wait (the landed-tile mbarrier), 1 A_work (next-tile bookkeeping, gather, radix 8, up to thread 0's arrival
    //   at the barrier), 2 A_bar (thread 0's arrival to the barrier's release), 3 B, 4 C+D (barrier to barrier),
    //   8 E up to thread 0's arrival, 7 E_bar (arrival to release);
    // and lane 0 of every warp adds its own time in E to 5 and the slowest warp's, per tile, to 6.
    // Compiled out by default.
#ifdef R8BGPU_PHASE_TIMERS
    __shared__ unsigned long long s_emax[2];
    if (ht == 0) s_emax[h] = 0;
    long long t_prev = clock64();
#define R8B_TICK(i)                                                                  \
    if (p.prof != nullptr && ht == 0) {                                              \
        const long long t_now = clock64();                                           \
        atomicAdd(&p.prof[i], (unsigned long long) (t_now - t_prev));                \
        t_prev = t_now;                                                              \
    }
#else
#define R8B_TICK(i)
#endif
    for (; u < n_units; u += stride) {
        // the tile after this one: its input starts moving towards L2 now
        Tile tn = t;
        int pathn = -1;
        if (u + stride < n_units) {
            tn = tile_of(p, u + stride);
            pathn = tile_input_path(src, tn);
            if (pathn == 2 && !tma_in) pathn = 1;
            if ((pathn == 1 || pathn == 2) && ht == 0) bulk_prefetch_l2(reinterpret_cast<const void*>(reinterpret_cast<unsigned long long>(tile_src(tn)) & ~15ull),
                                                        FM * sizeof(double));
        }
        // A. input -> registers -> radix-8 pass into the lower half of the buffer
        {
            double2 v[8];
            if (path == 2) {
                R8B_TICK(1)
                mbar_wait(&mb[1 + h], par_in);
                R8B_TICK(0)
                par_in ^= 1;
                const double2* st = buf + STAGE_UP;
#pragma unroll
                for (int j = 0; j < 8; j++) v[j] = st[ht + 256 * j];
            } else {
                gather_tile(v, src, t, path, ht);
            }
            fwd_pass1_r8(v, buf, tw2, twf, ht);
        }
        // a tile index past the call's table: the tile computes its own entry
        if (!COPY && u - t.ch * p.n_tiles >= p.n_tab && ht == HT - 1) s_te[h] = tile_entry(p, dst.base, u - t.ch * p.n_tiles);
        R8B_TICK(1)
        bar_half(h);
        R8B_TICK(2)
        // B. the two radix-16 passes act on 256-point blocks owned by one half-warp each
        constexpr bool fuse_c = (UP == 2); // the 1x pair keeps its separate split pass
        if (ht < FN / 16) {
            fwd_pass<256>(buf, tw2, ht);
            __syncwarp();
            if constexpr (fuse_c) fwd_pass16_skew(buf, ht);
            else fwd_pass<16>(buf, tw2, ht);
        }
        bar_half(h);
        R8B_TICK(3)
        // C. split + multiply by the filter spectrum -- fused into the first inverse pass (UP == 2), or in place
        if constexpr (fuse_c) {
            double2 z1[8], z2[8];
            cd1_load(buf, ht, z1, z2);
            bar_half(h);
            // this thread's W_M^kappa_0 and phi_g: 8 KB read by every tile, so they stay in L1 (held in registers for the
            // whole kernel, or loaded before the barrier, they cost 130-200 bytes of spills)
            if constexpr (CS) cd1s_compute(scs, __ldg(&p.cs_tab[CS_PAIRS + ht]), __ldg(&p.cs_tab[CS_PAIRS + HT + ht]), buf, ht, z1, z2);
            else cd1_compute(p, buf, ht, z1, z2);
        } else {
            double2 z1[4], z2[4], ze = make_double2(0.0, 0.0);
            c_load(buf, ht, z1, z2);
            if (ht == 0) ze = buf[fft_pad(slot_of<FN>(FN / 2))];
            bar_half(h);
#pragma unroll
            for (int i = 0; i < 4; i++) c1_pair_tab(p, buf, ht, i, z1[i], z2[i]);
            if (ht == 0) c1_pair_mid(p, buf, ze);
            bar_half(h);
        }
        // D. inverse transform
        if constexpr (UP == 2) {
            __syncwarp(); // the first inverse pass ran inside phase C (cd1_compute)
            inv_pass<256>(buf, tw2, ht);
            bar_half(h);
            {
                double2 v[16];
                inv3_load(buf, tw2, twf, ht, v);
                bar_half(h);
                y_store<PADV>(buf, v, ht, t.w, p.ysh);
            }
        } else {
            if (ht < FN / 16) {
                inv_pass<16>(buf, tw2, ht);
                __syncwarp();
                inv_pass<256>(buf, tw2, ht);
            }
            bar_half(h);
            {
                double2 v[8];
                inv1_last_load(buf, tw2, twf, ht, v);
                bar_half(h);
                y_store1<PADV>(buf, v, ht, t.w, p.ysh);
            }
        }
        bar_half(h);
        R8B_TICK(4)
        // E. interpolation out of shared memory
        if (pingpong) {
            mbar_wait(&mb[3 + h], par_turn);
            par_turn ^= 1;
        }
#ifdef R8BGPU_PHASE_TIMERS
        const long long t_e0 = clock64();
#endif
        {
            const double* yb = reinterpret_cast<const double*>(buf);
            const int ti = u - t.ch * p.n_tiles;
            const TileEntry& te = ti < p.n_tab ? tab[ti] : s_te[h];
            const int* si = te.s;
            const long long drow = (long long) t.ch * dst.stride; // the channel's row of the destination
            if constexpr (POLY) {
                // A warp takes 32 consecutive outputs per round: every lane evaluates ONE position (the timing expression costs a
                // double division), the four blocks of 8 read their rows' values by shuffle.  When all four blocks sit on the
                // same pair of bank rows -- 32 outputs drift ~1.15 rows, so mostly -- their DMMA chains are interleaved (four
                // independent accumulators hide the dependent-issue latency); otherwise block by block.
                const int ka = si[0], kb = si[1], N = p.poly_n, flen = p.flen, ksteps = (flen + 3) >> 2;
                const int row = lane >> 2, kq = lane & 3;
                const unsigned full = 0xffffffffu;
                const int n_rounds = (kb - ka + 31) >> 5;
                int cached_row = -2;
                double bq[8]; // B fragment of every K-step for the cached row pair (flen <= 32)
                auto load_b = [&](int fmin) { // column n = lane/4: component n>>1 of row fmin + (n&1); columns 6, 7 unused
                    cached_row = fmin;
                    int brow = fmin + (row & 1);
                    if (brow > p.fracs) brow = p.fracs;
                    const double* __restrict__ br = p.bank + (long long) brow * 3 * flen + (row >> 1);
#pragma unroll
                    for (int ks = 0; ks < 8; ks++) {
                        const int tap = 4 * ks + kq;
                        bq[ks] = (ks < ksteps && tap < flen && row < 6) ? __ldg(br + 3 * tap) : 0.0;
                    }
                };
                for (int rd = wh; rd < n_rounds; rd += HT / 32) {
                    const int k_own = ka + 32 * rd + lane;
                    const bool v_own = k_own < kb;
                    long long ip;
                    double fpos;
                    poly_position(p, v_own ? k_own : kb - 1, ip, fpos);
                    double x_own = __dmul_rn(fpos, (double) p.fracs);
                    const int f_own = __double2int_rz(x_own);
                    x_own = __dsub_rn(x_own, (double) f_own);
                    const int y_own = (int) (ip - p.fll - 2 * t.w);
                    int fm = v_own ? f_own : 0x7fffffff; // min row of the lane's block of 8 outputs
                    fm = min(fm, __shfl_xor_sync(full, fm, 1));
                    fm = min(fm, __shfl_xor_sync(full, fm, 2));
                    fm = min(fm, __shfl_xor_sync(full, fm, 4));
                    // per block q: this lane's row (lane 8q + row of the round)
                    int yi[4], fr[4], ya0[4], fmin[4];
                    bool vr[4], fast[4];
                    bool all_fast = true;
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const int srcl = 8 * q + row;
                        yi[q] = __shfl_sync(full, y_own, srcl);
                        fr[q] = __shfl_sync(full, f_own, srcl);
                        vr[q] = __shfl_sync(full, (int) v_own, srcl) != 0;
                        ya0[q] = __shfl_sync(full, y_own, 8 * q);
                        fmin[q] = __shfl_sync(full, fm, 8 * q);
                        const bool blk_live = __shfl_sync(full, (int) v_own, 8 * q) != 0; // block has at least one output
                        const bool fits = !vr[q] || (yi[q] == ya0[q] + N * row && fr[q] - fmin[q] <= 1);
                        fast[q] = blk_live && __all_sync(full, fits) && ya0[q] >= 0 && ya0[q] + 7 * N + 4 * ksteps <= p.ylen;
                        all_fast = all_fast && (fast[q] || !blk_live);
                    }
                    // do the live blocks share block 0's row pair?
                    bool same = all_fast;
#pragma unroll
                    for (int q = 1; q < 4; q++) {
                        const bool blk_live = __shfl_sync(full, (int) v_own, 8 * q) != 0;
                        if (blk_live) {
                            const bool in_pair = !vr[q] || (fr[q] - fmin[0] >= 0 && fr[q] - fmin[0] <= 1);
                            same = same && __all_sync(full, in_pair);
                        }
                    }
                    double res[4] = {0.0, 0.0, 0.0, 0.0}; // output of (block q, this lane's row), meaningful in lanes kq == 0
                    if (same) {
                        if (fmin[0] != cached_row) load_b(fmin[0]);
                        double c0[4] = {0.0, 0.0, 0.0, 0.0}, c1[4] = {0.0, 0.0, 0.0, 0.0};
                        const double* ya[4];
#pragma unroll
                        for (int q = 0; q < 4; q++) ya[q] = yb + (fast[q] ? ya0[q] : 0) + N * row + kq;
#pragma unroll
                        for (int ks = 0; ks < 8; ks++)
                            if (ks < ksteps) {
#pragma unroll
                                for (int q = 0; q < 4; q++) dmma884(c0[q], c1[q], ya[q][4 * ks], bq[ks]);
                            }
#pragma unroll
                        for (int q = 0; q < 4; q++) res[q] = (fr[q] - fmin[0]) ? c1[q] : c0[q];
                    } else {
#pragma unroll
                        for (int q = 0; q < 4; q++) {
                            if (!fast[q]) continue; // (warp-uniform)
                            if (fmin[q] != cached_row) load_b(fmin[q]);
                            double c0 = 0.0, c1 = 0.0;
                            const double* yq = yb + ya0[q] + N * row + kq;
#pragma unroll
                            for (int ks = 0; ks < 8; ks++)
                                if (ks < ksteps) dmma884(c0, c1, yq[4 * ks], bq[ks]);
                            res[q] = (fr[q] - fmin[q]) ? c1 : c0;
                        }
                    }
                    // combine the three components of every row: lanes kq = 0, 1, 2 hold D0, D1, D2
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const double xr = __shfl_sync(full, x_own, 8 * q + row);
                        const double d1 = __shfl_sync(full, res[q], (lane & ~3) + 1), d2 = __shfl_sync(full, res[q], (lane & ~3) + 2);
                        double outv = fma(__dmul_rn(xr, xr), d2, fma(xr, d1, res[q]));
                        const bool slow = vr[q] && !(same || fast[q]);
                        if (slow && kq == 0 && yi[q] >= 0 && yi[q] + flen <= p.ylen) {
                            // one output, the reference's own order: c = c0 + c1 x + c2 x^2 per tap, taps ascending
                            const double x2 = __dmul_rn(xr, xr);
                            const double* __restrict__ br = p.bank + (long long) fr[q] * 3 * flen;
                            outv = 0.0;
                            for (int i = 0; i < flen; i++)
                                outv = fma(fma(__ldg(br + 3 * i + 2), x2, fma(__ldg(br + 3 * i + 1), xr, __ldg(br + 3 * i))), yb[yi[q] + i], outv);
                        }
                        if (vr[q] && kq == 0) dst_write_f(dst, t.ch, p.e0 + ka + 32 * rd + 8 * q + row, outv);
                    }
                }
            } else if constexpr (COPY) {
                // owned positions [A0, A1) clipped to this call's range; position q sits at y index q - 2 w
                long long q0 = t.A0 > p.e0 ? t.A0 : p.e0, q1 = t.A1 < p.e1 ? t.A1 : p.e1;
                const int off = (int) (q0 - 2 * t.w), cnt = q1 > q0 ? (int) (q1 - q0) : 0;
                double* const orow = dst.ptr + (long long) t.ch * dst.stride;
                const long long d0 = q0 - dst.base;
                const bool pair_ok = ((off | (int) (d0 & 1)) & 1) == 0 && (reinterpret_cast<unsigned long long>(orow) & 15) == 0;
                if (pair_ok) { // even start on both sides: 16-byte moves (a pair never straddles the ring's end)
                    for (int i = 2 * ht; i + 1 < cnt; i += 2 * HT)
                        *reinterpret_cast<double2*>(orow + ((d0 + i) & dst.mask)) = *reinterpret_cast<const double2*>(yb + off + i);
                    if ((cnt & 1) && ht == 0) orow[(d0 + cnt - 1) & dst.mask] = yb[off + cnt - 1];
                } else {
                    for (int i = ht; i < cnt; i += HT) orow[(d0 + i) & dst.mask] = yb[off + i];
                }
            } else if constexpr (TC) {
                MmaTile mt;
                mt.load(te, drow);
                const int n_mu = mt.n_j > 0 ? mma_units(p, mt.c_cnt) : 0, smaxp = p.smaxp;
                double* const so = dst.ptr + drow + (te.off & dst.mask);
                constexpr int WS = HT / 32;
                // MB = M tiles (pairs of blocks) per unit, a per-call choice (p.mbu)
                auto run_units = [&](auto mb_tag) {
                    constexpr int MB = decltype(mb_tag)::value;
                    MmaUnit mu;
                    mu.set(wh, n_groups);
                    for (int unit = wh; unit < n_mu; unit += WS) {
                        int yo[2 * MB];
                        const int goff = s_goff[mu.g];
#pragma unroll
                        for (int i = 0; i < 2 * MB; i++) yo[i] = mma_a_index(p, mt, mu, goff, i, lane);
                        const double* const gb = sbank + mma_b_index(p, mu, lane);
                        double acc[MB][4];
#pragma unroll
                        for (int m = 0; m < MB; m++) acc[m][0] = acc[m][1] = acc[m][2] = acc[m][3] = 0.0;
                        auto kchunk = [&](auto kw_tag, int k0) {
                            constexpr int KW = decltype(kw_tag)::value;
                            double b[KW / 4];
#pragma unroll
                            for (int i = 0; i < KW / 4; i++) b[i] = gb[8 * k0 + 32 * i];
#pragma unroll
                            for (int m = 0; m < MB; m++) {
                                double a[KW / 2];
#pragma unroll
                                for (int i = 0; i < KW / 2; i++) {
                                    const int yi = yo[2 * m + (i & 1)] + k0 + 4 * (i >> 1);
                                    a[i] = PADV ? yb[ylay(yi, p.ysh)] : yb[yi];
                                }
                                dmma16<KW>(acc[m], a, b);
                            }
                        };
                        using K16 = std::integral_constant<int, 16>;
                        const int k16 = smaxp & ~15;
#pragma unroll 1
                        for (int k0 = 0; k0 < k16; k0 += 16) kchunk(K16(), k0);
                        if (smaxp & 8) kchunk(std::integral_constant<int, 8>(), k16);
                        if (smaxp & 4) kchunk(std::integral_constant<int, 4>(), k16 + (smaxp & 8));
#pragma unroll
                        for (int m = 0; m < MB; m++) {
                            mma_store<LIN>(p, dst, t.ch, mt, so, mu, 2 * m, lane, acc[m][0], acc[m][1]);
                            mma_store<LIN>(p, dst, t.ch, mt, so, mu, 2 * m + 1, lane, acc[m][2], acc[m][3]);
                        }
                        mu.advance(WS, n_groups);
                    }
                };
                switch (mma_mbu(p)) {
                case 2: run_units(std::integral_constant<int, 1>()); break;
                case 4: run_units(std::integral_constant<int, 2>()); break;
                default: run_units(std::integral_constant<int, 3>()); break;
                }
            } else if (si[0] > 0) {
                const int n_tasks = TaskGeom<IRV, GLOG>::n_tasks(p, si[1]);
                double* const stg = p.stage_off > 0 ? reinterpret_cast<double*>(smem) + p.stage_off + (tid >> 5) * 256 : nullptr;
                double* const so = dst.ptr + drow + (te.off & dst.mask);
                for (int task = wh; task < n_tasks; task += HT / 32) {
                    TaskGeom<IRV, GLOG> g;
                    g.set(p, s_goff, task, lane);
                    int yo[IQ2];
                    interp_windows<IRV, GLOG>(p, g, si, yo);
                    double acc[IRV][IQ2];
                    interp_acc<IRV, PADV>(yb, sbank + g.grp * esz, yo, p.smaxp, p.ysh, acc);
                    if (IRV == 8 && dst.mask == -1 && stg != nullptr) {
                        if constexpr (IRV == 8) interp_store_staged<GLOG>(p, si, so, stg, task, lane, acc);
                    } else {
                        interp_store_direct<IRV, GLOG>(p, dst, t.ch, g, si, so, acc);
                    }
                }
            }
        }
#ifdef R8BGPU_PHASE_TIMERS
        if (p.prof != nullptr && lane == 0) {
            const unsigned long long dt = (unsigned long long) (clock64() - t_e0);
            atomicAdd(&p.prof[5], dt);
            atomicMax(&s_emax[h], dt);
        }
#endif
        R8B_TICK(8)
        bar_half(h); // the buffer is free again
        R8B_TICK(7)
#ifdef R8BGPU_PHASE_TIMERS
        if (p.prof != nullptr && ht == 0) {
            atomicAdd(&p.prof[6], s_emax[h]);
            s_emax[h] = 0;
        }
#endif
        if (ht == 0) {
            if (pingpong) mbar_arrive(&mb[4 - h]);
            if (pathn == 2) {
                fence_proxy_async(); // generic-proxy reads of the buffer are ordered before the async-proxy write
                mbar_expect_tx(&mb[1 + h], FM * sizeof(double));
                bulk_g2s(buf + STAGE_UP, tile_src(tn), FM * sizeof(double), &mb[1 + h]);
            }
        }
        t = tn;
        path = pathn;
    }
#undef R8B_TICK
}

template <int IRV, bool PADV, int GLOG, bool TC = false, int UP = 2, bool COPY = false, bool POLY = false, bool CS = false,
          bool LIN = false>
static void launch_inst2(const FusedParams& p, const SrcView& src, const DstView& dst, int grid, int smem, cudaStream_t st,
                         FusedVariant* v)
{
    ensure_dyn_smem<k_up2_frac2<IRV, PADV, GLOG, TC, UP, COPY, POLY, CS, LIN>>(227 * 1024);
    k_up2_frac2<IRV, PADV, GLOG, TC, UP, COPY, POLY, CS, LIN><<<(unsigned) grid, NT2, smem, st>>>(p, src, dst);
    if (v != nullptr) {
        *v = FusedVariant();
        v->kernel = 2;
        v->ir = IRV;
        v->pad = PADV;
        v->glog = GLOG;
        v->tc = TC;
        v->up = UP;
        v->copy = COPY;
        v->poly = POLY;
        v->cs = CS;
        v->lin = LIN;
        v->mbu = p.mbu;
    }
}

// the tensor-path interpolation of a whole-stepping pair, with the stores specialised for a linear fp64 destination
template <bool PADV, int UP, bool CS>
static void launch_tc(const FusedParams& p, const SrcView& src, const DstView& dst, int grid, int smem, cudaStream_t st,
                      FusedVariant* v)
{
    if (dst.fmt == FMT_F64 && dst.mask == -1) launch_inst2<8, PADV, 0, true, UP, false, false, CS, true>(p, src, dst, grid, smem, st, v);
    else launch_inst2<8, PADV, 0, true, UP, false, false, CS>(p, src, dst, grid, smem, st, v);
}

template <bool CS>
static void launch_f2(const FusedParams& p, const SrcView& src, const DstView& dst, int grid, int smem, cudaStream_t st,
                      FusedVariant* v)
{
    const bool pad = p.ysh != 31;
#define R8B_F2_CASE(IRV, GL)                                                              \
    if (pad) launch_inst2<IRV, true, GL, false, 2, false, false, CS>(p, src, dst, grid, smem, st, v); \
    else launch_inst2<IRV, false, GL, false, 2, false, false, CS>(p, src, dst, grid, smem, st, v);
    if (p.mode == 1) { // order-2 bank on the tensor path (ratios close to an integer; plain y layout)
        launch_inst2<8, false, 0, true, 2, false, true, CS>(p, src, dst, grid, smem, st, v);
        return;
    }
    if (p.mode == 2) { // BlockConvolver 2/1 alone
        launch_inst2<8, false, 0, true, 2, true, false, CS>(p, src, dst, grid, smem, st, v);
        return;
    }
    if (p.up == 1) { // batch_create only routes a 1x pair here when the tensor-path bank fits
        if constexpr (!CS) {
            if (pad) launch_tc<true, 1, false>(p, src, dst, grid, smem, st, v);
            else launch_tc<false, 1, false>(p, src, dst, grid, smem, st, v);
        }
    } else if (p.ir == 8 && (p.flags & 4)) {
        if (pad) launch_tc<true, 2, CS>(p, src, dst, grid, smem, st, v);
        else launch_tc<false, 2, CS>(p, src, dst, grid, smem, st, v);
    } else if (p.ir == 10) {
        if (p.glog == 2) { R8B_F2_CASE(10, 2) } else if (p.glog == 1) { R8B_F2_CASE(10, 1) } else { R8B_F2_CASE(10, 0) }
    } else {
        if (p.glog == 2) { R8B_F2_CASE(8, 2) } else if (p.glog == 1) { R8B_F2_CASE(8, 1) } else { R8B_F2_CASE(8, 0) }
    }
#undef R8B_F2_CASE
}

// p.n_ch, p.n_tiles, p.span ... describe the call; n_sm = SMs of the device (persistent grid).
void launch_up2_frac2(const FusedParams& p, const SrcView& src, const DstView& dst, int n_sm, cudaStream_t st, FusedVariant* v)
{
    const int n_units = p.n_tiles * p.n_ch;
    if (n_units <= 0) return;
    int grid = (n_units + 1) / 2;
    if (grid > n_sm) grid = n_sm;
    const bool cs = p.up != 1 && p.cs_tab != nullptr;
    // the tile table takes what the plan leaves of shared memory: every tile index of the call where it fits
    // (a 65536-sample block needs about 20 entries of 24 bytes), the first n_tab otherwise
    FusedParams q = p;
    int smem = fused2_smem_bytes(p.gbank_smem_len, cs, p.stage_off > 0);
    q.tab_off = smem;
    q.n_tab = p.mode == 2 ? 0 : std::max(0, std::min(p.n_tiles, (kFused2SmemMax - smem) / (int) sizeof(TileEntry)));
    smem += q.n_tab * (int) sizeof(TileEntry);
    if (cs) launch_f2<true>(q, src, dst, grid, smem, st, v);
    else launch_f2<false>(q, src, dst, grid, smem, st, v);
}

} // namespace r8bgpu

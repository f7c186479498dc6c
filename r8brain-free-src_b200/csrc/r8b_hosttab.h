// r8b_hosttab.h -- host-side tables and tile geometry of the device kernels, shared by the engine
// (r8b_capi.cu) and by the CPU emulation of the fused kernel that the tests run without a GPU
// (tests/cpp/fused2_emul.cu).  Nothing here touches the device.
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "r8b_kernels.h"
#include "r8b_plan.h"

namespace r8bgpu {

// Low-pass spectrum of a BlockConvolver stage (CDSPFIRFilter.h:492-520 as arithmetic: direct long-double DFT of
// the designed taps, polyphase-packed g_0 + i g_1 for 2x stages, pre-scaled by 1/M resp. 1/(2M)) in FFT slot order,
// and the twiddle table exp(-2 pi i k / M).
void build_spectrum(const StageDesc& s, int fft_log2, std::vector<double2>& spec_slots, std::vector<double2>& tw,
                    double* nyq_gain);

// The same for the large-tile path (fft_log2 14..16, r8b_bclarge.cuh): spectrum of the whole kernel h with U = 1 (2x
// stages run on the zero-stuffed view), pre-scaled by 1/M, in the slot order (k % R0) * 4096 + slot_of<4096>(k / R0);
// tw4096 = exp(-2 pi i k / 4096), tw_m = exp(-2 pi i k / M).  h is real, so H[M - k] = conj H[k] and only half the
// bins are summed (and only the kept 1/D of them for reference-exact decimation).
void build_spectrum_large(const StageDesc& s, int fft_log2, std::vector<double2>& spec_slots, std::vector<double2>& tw4096,
                          std::vector<double2>& tw_m, double* nyq_gain);

// Tile length of an overlap-save stage: the b in [min_log2, max_log2] that minimises b * 2^b / (2^b - 2 lg) with at
// least 64 valid positions per tile; -1 when none has.  R8BGPU_FFT_LOG2 forces a length inside the range.
int choose_fft_log2(int lg, int min_log2, int max_log2);

// How a BlockConvolver stage runs, before the fusion decisions of batch_create (which may move it to a fused kernel).
struct BcTile {
    int fft_log2 = -1;  // log2 of the tile length M; -1: no supported tile
    int lg = 0;         // half support of the filter as seen from one tile sample
    int virt_up = 1;    // > 1: a 1x convolution over the zero-stuffed view of the source (x[t / virt_up] where virt_up | t)
    int up = 1;         // up-factor of the tile operator: 2 (polyphase k_blockconv) or 1
    bool large = false; // M >= 16384: the large-tile path (r8b_bclarge.cuh)
};
// allow_large = false: the rule of the in-shared-memory tiles alone (1x stages up to 8192 points, 2x up to 4096,
// reference-exact decimation on the reference's own block of 64 .. 8192 points).  With allow_large the large-tile path
// takes exactly the stages that rule refuses, with M from {16384, 32768, 65536}.
BcTile blockconv_tile(const StageDesc& s, bool allow_large = true);

// Per-call tile geometry of an unfused BlockConvolver (k_blockconv and the large-tile path) for the outputs [e0, e1):
// every field of p except nyq_gain, spec and tw (left zero).
void blockconv_call_fields(BlockConvParams& p, const StageDesc& s, int virt_up, int lg, int fft_log2, long long e0, long long e1);

// [q][r] twiddle tables of the fused kernels: 256 entries W_256^(r q), then 256 entries W_4096^(r q)
std::vector<double2> build_tw_tab(const std::vector<double2>& tw4096);
// phase C operands of the v2 fused kernel's 1x pair in thread order (FusedParams::c_tab, the layout c1_pair_tab() reads);
// empty for up = 2, whose phase C runs inside the first inverse pass (build_cd_tab)
std::vector<double2> build_c_tab(const std::vector<double2>& spec_slots4096, const std::vector<double2>& tw4096, int up);

// "2x BlockConvolver -> FracInterpolator" pair: margins and span of the M = 4096 tiles
struct FusedGeom {
    bool ok = false;
    int lg = 0, yl = 0, yr = 0, span_max = 0, ysh = 31;
    int up = 2; // up-factor of the BlockConvolver: 2, or 1 (v2 kernel with the tensor-path interpolation only)
};
FusedGeom fused_geometry(const StageDesc& bc, const StageDesc& frac);

// Whole-stepping bank re-laid for the fused kernels: for EVERY first phase r0 a [smaxp][ir] block holding the
// filters of phases r0..r0+ir-1 pre-shifted by their window offsets and zero-padded (CDSPFracInterpolator.h:991-1060
// reads bank[(j*InStep) % OutStep] at window floor(j*InStep/OutStep)).
struct GroupBank {
    int ir = 8, smaxp = 0, n_groups = 0;
    std::vector<double> gb;   // [out_step][smaxp][ir]
    std::vector<int> go;      // [out_step] floor(r0*in_step/out_step)
    std::vector<int> off, row; // per phase: window offset, bank row
};
int choose_group_ir(const StageDesc& frac);
// operands of the v2 kernel's fused phase C + first inverse pass (FusedParams::cd_tab)
std::vector<double2> build_cd_tab(const std::vector<double2>& spec_slots4096, const std::vector<double2>& tw4096);
// the same spectrum in its symmetric half-size form (FusedParams::cs_tab, r8b_fused2_core.cuh cs_entry): (a0[k], a1[k]) for
// k = 0..2048 in thread order, then per thread W_M^kappa_0 and phi_g; of the 2x BlockConvolver stage s (M = 4096)
std::vector<double2> build_cs_tab(const StageDesc& s, const std::vector<double2>& tw4096);
// The largest phase-group bank k_up2_frac2 may hold in shared memory for interpolator stage f (either bank layout; 0 when
// f has none), and whether the symmetric spectrum table fits beside a bank of that size.  Decided once per plan, so every
// variant of the kernel (tensor-path or FMA interpolation, staging or none) runs the same phase-C arithmetic.
int fused2_bank_doubles_max(const StageDesc& f);
bool fused2_cs_fits(int bank_doubles_max);
// the same for the round-1 fused kernel (tile pairs, 512 threads): [u < 4][item < 2][tid < 512] = spectrum at the slot
// s1 = 16*((tid>>3) + 64u) + (tid&7) and at the slot of the mirrored frequency
std::vector<double2> build_c_tab_v1(const std::vector<double2>& spec_slots4096);

// frag_order (ir == 8 only): within every block of 4 taps the 32 values are stored as [phase][tap % 4] -- the B-fragment
// order of mma.sync m8n8k4, so a warp's load of one K-step is 256 contiguous bytes
GroupBank build_group_bank(const StageDesc& frac, int ir, bool frag_order = false);

// Whole-stepping call: the fields of FusedParams that follow from the interpolator stage and this call's output
// range [e0, e1) alone (positions are indices of the 2x-rate stream; p_lo even).
void fused_whole_fields(FusedParams& p, const StageDesc& frac, long long e0, long long e1);

// Per-call tile geometry of the v2 fused kernel (one tile per half-CTA): fills p.p_lo (input: first needed position,
// even), p.n_tiles, p.span.  cur_parity >= 0: parity of the caller's block base index, so that FFT windows start on
// 16-byte boundaries of the block (bulk-copied input tiles); -1: no constraint.
void fused2_tiles(FusedParams& p, const FusedGeom& g, int cur_parity);

// The settings the lock-step launch path reads for a fused order-2 pair, on every call.
struct PolyKnobs {
    bool bank_global = false; // R8BGPU_BANK_GLOBAL: no bank rows staged in shared memory
    bool single = false;      // R8BGPU_POLY_SINGLE: one output per thread (poly_n 0)
};
PolyKnobs poly_knobs_env();

// How one lock-step call runs a 2x BlockConvolver fused with the order-2 interpolator behind it.  The kernel's
// bookkeeping (r8b_poly.cuh) reads these fields of FusedParams; r8b_capi.cu copies them in and
// r8bgpu_plan_order2_info reports them.
struct PolyCall {
    bool v2 = false;           // the call runs on k_up2_frac2 (the plan's R8BGPU_POLY_V2 opt-in, a ratio within 1e-3 of 1..3)
    int n_tiles = 0, span = 0; // tiles of the call and the positions each owns (k_up2_frac: processed in pairs)
    long long p_lo = 0;        // first owned position (k_up2_frac2 may move it back one sample pair)
    int poly_dir = 0;          // +1 / -1: a run of bank rows ascending / descending with k is staged; 0: none
    int poly_rows_cap = 0;     // rows the staged run may hold
    int poly_row_stride = 0;   // doubles between staged rows
    int poly_chunks = 1;       // pieces of a pair's outputs, each with its own run
    int poly_n = 0;            // 1..3: four consecutive outputs per thread, windows ~poly_n apart (poly_block4<poly_n>)
    int ysh = 31;              // y layout of the tile buffers (4: padded, 31: plain)
    int smem_bytes = 0;        // dynamic shared memory of the launch (k_up2_frac only; 0 on k_up2_frac2)
};
// f: the order-2 interpolator behind a fused 2x BlockConvolver of geometry g; f2_poly: the plan may run the pair on
// k_up2_frac2 (FusedPlan::poly_v2); ssr / dsr: the call's rates (a trim factor moves dsr); [p_lo, p_hi): the call's owned
// positions (p_lo even); cur_parity as for fused2_tiles.
PolyCall plan_poly_call(const StageDesc& f, const FusedGeom& g, bool f2_poly, double ssr, double dsr, long long p_lo,
                        long long p_hi, int cur_parity, const PolyKnobs& k);
int fused2_choose_glog(int span, int in_step, int out_step, int ir);
// blocks of 8 stepping cycles per work unit of the tensor-path interpolation: fewest (rounds over a half's 8 warps) x blocks
int fused2_choose_mbu(int span, int in_step, int out_step);

} // namespace r8bgpu

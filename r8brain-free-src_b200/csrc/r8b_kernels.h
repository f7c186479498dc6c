// r8b_kernels.h -- launch interface between the host engine (r8b_engine.cu) and the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cmath>

namespace r8bgpu {

// Opt a kernel into more than 48 KB of dynamic shared memory, once per (kernel, device): thread-safe, and
// devices beyond the bitmap simply set the attribute on every launch.
template <auto Kernel>
inline void ensure_dyn_smem(int bytes)
{
    static std::atomic<unsigned long long> done[4];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 256 && ((done[dev >> 6].load(std::memory_order_acquire) >> (dev & 63)) & 1ull)) return;
    // the opt-in limit (227 KB per CTA on sm_90) covers static + dynamic shared memory together
    cudaFuncAttributes fa{};
    if (cudaFuncGetAttributes(&fa, Kernel) == cudaSuccess && bytes > 227 * 1024 - (int) fa.sharedSizeBytes)
        bytes = 227 * 1024 - (int) fa.sharedSizeBytes;
    if (cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) {
        cudaGetLastError();
        return; // not marked done: the launch reports the error
    }
    if (dev >= 0 && dev < 256) done[dev >> 6].fetch_or(1ull << (dev & 63), std::memory_order_release);
}

// caller-side sample formats (values of r8bgpu_sample_format, include/r8bgpu.h)
enum { FMT_F64 = 0, FMT_F32 = 1, FMT_S16 = 2, FMT_S24 = 3, FMT_S32 = 4, FMT_U8 = 5, FMT_ULAW = 6, FMT_ALAW = 7,
       FMT_DSD_LSB = 16, FMT_DSD_MSB = 17 };

// A per-channel sample stream addressed by ABSOLUTE sample index n (n = 0 is the first sample
// after clear()).  Samples with n >= cur_base are read from the caller's block of this
// process() call; older samples come from a power-of-two ring that holds the recent past.
// Indices < 0 land in ring slots that are still zero (rings are cleared at clear()).
struct SrcView {
    const double* ring;    // [n_ch][ring_stride]
    long long ring_stride;
    long long ring_mask;   // capacity-1
    const double* cur;     // [n_ch][cur_stride] or nullptr
    long long cur_stride;
    long long cur_base;    // absolute index of cur[0]; LLONG_MAX when there is no cur block
    long long avail;       // samples with n >= avail do not exist yet (read as 0)
    // Caller-side sample format of the cur block (FMT_*; FMT_F64 = plain doubles).  Only the v2 fused kernel and the
    // history copy read typed blocks: cur then points at planar samples of that format, cur_stride counts samples, and
    // a value is (double) sample * cur_scale -- the conversion of CDSPResampler::oneshot<Tin,Tout>()
    // (CDSPResampler.h:592-651) done in the gather instead of in a kernel of its own.  The half-band decimators
    // (k_hbdown, k_hbdown_cascade) and the history copy read planar DSD blocks the same way (r8b_dsd.cuh): cur then
    // points at bytes, cur_stride counts bytes, and sample n is a bit of byte (n - cur_base) / 8.
    int cur_fmt = 0;
    double cur_scale = 1.0;
};

struct DitherCall;

// Destination stream: either a ring (mask = capacity-1, base = 0) or a linear block whose
// element 0 is absolute index `base` (mask = -1).
struct DstView {
    double* ptr;           // [n_ch][stride]
    long long stride;
    long long mask;
    long long base;
    // Sample format of a LINEAR destination (the v2 fused kernel's tensor-path stores only): ptr then addresses planar
    // samples of that format, stride counts samples, and a stored value is (T) (y * scale).
    int fmt = 0;
    double scale = 1.0;
    // flat TPDF in those stores (r8b_dither.cuh): the batch's tables, and the batch channel of this launch's channel 0
    const DitherCall* dither = nullptr;
    int dither_ch0 = 0;
};

// Ragged calls (channels with schedules of their own): one record per channel and stage holds what differs between
// channels; the kernels' RAG instantiations read these fields from rr[channel] instead of the uniform parameters, whose
// ranges then describe the largest channel (grid size).  A CTA past its channel's tile count exits at once.
struct RaggedRec {
    long long m0, m1;      // BlockConv: input-rate positions [m0, m1); history copy: samples [m0, m1) to keep
    long long e0, e1;      // output indices to write
    long long cur_base, avail; // this channel's source view (SrcView fields of the same name)
    long long dst_base;    // linear destination: absolute index of element 0
    long long p0;          // order-2 interpolator timing state at the first output (FracParams fields)
    double in_pos_shift, fpos0;
    double ssr, dsr;       // order-2 interpolator: this channel's rates (a trim plan's per-channel dsr)
    int in_counter0, in_pos_int0;
    int n_tiles, adv;      // BlockConv tiles (and advance per tile)
};

struct BlockConvParams {
    int up, down;          // up is 1 or 2 here; other up-factors run as up = 1 on a zero-stuffed view
    int src_up;            // > 1: tile positions index the zero-stuffed stream x[t/src_up] (t % src_up == 0)
    int lg;                // half support of the polyphase filters, in input samples
    int fft_log2;          // log2(M)
    int adv;               // valid input-rate positions per tile (<= M - 2*lg)
    long long m0, m1;      // input-rate positions [m0,m1) whose outputs may be needed
    long long e0, e1;      // output indices to write
    int n_tiles;
    int trunc;             // 0, or D for reference-exact power-of-two decimation (see k_blockconv)
    double nyq_gain;       // scaled filter response at bin M/(2D) (trunc only)
    const double2* spec;   // filter spectrum in slot order, pre-scaled (device)
    const double2* tw;     // twiddles exp(-2*pi*i*k/M) (device)
};

struct FracParams {
    int flen, fll;
    long long e0, e1;
    const double* bank;    // device; [(fracs+1)][flen][order+1]
    // whole stepping
    int in_step, out_step;
    // polynomial (order 2)
    int fracs;
    double ssr, dsr;
    int in_counter0, in_pos_int0;
    double in_pos_shift, fpos0;
    long long p0;
    const int* pos_dp;       // R8B_FASTTIMING: per-output position - p0 and fraction (else nullptr)
    const double* pos_fpos;
};

struct HbParams {
    int ntaps;
    long long e0, e1;
    double taps[14];
};

// Fused chain of up to 6 half-band 2x DOWNsamplers (k_hbdown_cascade): every intermediate rate lives in shared memory.
// Stream s is the input of stage s (stream 0 = the cascade's source, stream n_stages = its output).
struct HbDownCascParams {
    int n_stages;
    int ntaps[6];
    double taps[6][14];
    long long e0, e1;      // output indices of the LAST stage to write
    int w;                 // final outputs per tile
    int n_tiles;
    int back[7];           // stream-s samples needed below 2^(n-s) * m for final output m (back[n] = 0)
    int boff[7];           // offsets (doubles) of the per-stream buffers in dynamic shared memory: even half, then odd half
    int cap[7];            // doubles per half of stream s's buffer
};
int hbdown_cascade_plan(HbDownCascParams& p, int smem_budget_doubles); // fills w, back, boff, cap; returns smem bytes (0: does not fit)
void launch_hbdown_cascade(const HbDownCascParams& p, int smem_bytes, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st);

// Fused chain of up to 6 half-band 2x upsamplers (k_hbup_cascade).
struct HbCascadeParams {
    int n_stages;
    int ntaps[6];
    double taps[6][14];
    long long e0, e1;      // output indices of the LAST stage to write
    long long a0;          // first tile starts at this position of the cascade's input stream
    int w;                 // tile width in input-stream samples
    int n_tiles;
    int lo_off[7], hi_off[7]; // stage-k stream range a tile needs: [2^k*A - lo_off[k], 2^k*(A+w) + hi_off[k])
    int boff[7];           // offsets (doubles) of the per-stage buffers in dynamic shared memory
    int fuse_last2;        // stages c-2 and c-1 run as one pass (no buffer for stream c-1)
};
bool hb_last2_supported(int t1, int t2);
// From n_stages and ntaps: fills lo_off, hi_off, fuse_last2 (where allowed and instantiated), w and boff for a CTA of at
// most smem_budget_doubles; returns its shared-memory bytes.  e0, e1, a0 and n_tiles are the call's.
int hbup_cascade_plan(HbCascadeParams& p, int smem_budget_doubles, bool allow_last2);
void launch_hbup_cascade(const HbCascadeParams& p, int smem_bytes, const SrcView& src, const DstView& dst,
                         int n_ch, cudaStream_t st);

// Fused 2x BlockConvolver + fractional interpolator (r8b_fused.cu).  Positions are indices of the
// 2x-rate stream between the two stages.
struct FusedParams {
    int mode;              // 0 whole stepping, 1 order-2 bank, 2 (v2 kernel only) no interpolator: the 2x stream itself is the output
    int n_tiles;           // tiles of `span` owned positions each, processed in pairs
    int stage_off;         // offset (doubles) of the store staging area in dynamic smem, 0 = none
    int debug;             // profiling experiments only (R8BGPU_DEBUG): bit0 skip interp stores, bit1 skip tap loop
    unsigned long long* prof; // optional: 10 phase-cycle accumulators (R8BGPU_PROFILE), else nullptr
    int span;              // even
    long long p_lo, p_hi;  // owned position range of this call [p_lo, p_hi), p_lo even
    int yl;                // left margin of a tile's valid range (>= fll, even)
    int lg;                // half support of the polyphase low-pass, input samples
    int ysh;               // y layout: index i lives at i + (i >> ysh) (31 = plain)
    const double2* spec;   // low-pass spectrum, slot order, pre-scaled by 1/(2M)
    const double2* tw;     // exp(-2*pi*i*k/M)
    // interpolator
    const double* bank;
    int bank_len, bank_in_smem;
    int flen, fll;
    long long e0, e1;      // outputs of this call
    int in_step, out_step;
    const double* gbank;   // whole stepping: for EVERY first phase r0 in [0,out_step): [smaxp][ir] shifted, zero-padded taps
                           // of phases r0..r0+ir-1 (phases past out_step-1 continue in the next stepping cycle)
    int gbank_len, smaxp;  // doubles in gbank; padded window length (multiple of 4)
    int ir;                // phases per group (8)
    int gbank_smem_len;    // doubles of the per-call bank selection kept in shared memory (n_groups * smaxp * ir)
    int delta, wrap;       // first phase of group 0 (= e0 mod 8 when out_step % 8 == 0, else 0); wrap = rows may span cycles
    const int* goff;       // [out_step] floor(r0*in_step/out_step)
    const int* phase_off;  // [out_step] floor(r*in_step/out_step)
    const int* phase_row;  // [out_step] (r*in_step) % out_step
    int fracs;
    double ssr, dsr;
    int in_counter0, in_pos_int0;
    double in_pos_shift, fpos0;
    long long p0;
    const int* pos_dp;       // R8B_FASTTIMING tables (else nullptr)
    const double* pos_fpos;
    // order-2 bank: when the bank row index drifts slowly and monotonically (mod fracs) with the output index,
    // the rows a tile pair needs are a short circular run that is staged in shared memory
    int poly_dir;            // +1 rows ascend with k, -1 descend, 0 no staging
    int poly_rows_cap;       // rows of shared memory available for the run
    int poly_row_stride;     // doubles between staged rows: 3*flen padded so that consecutive rows start 4 (mod 8)
                             // banks apart -- lanes that sit on different rows then load without bank conflicts
    int poly_n;              // > 0: input positions advance by ~poly_n per output; threads take 4 consecutive outputs
    int poly_chunks;         // a pair's outputs are processed in this many pieces, each with its own run (>= 1)
    // v2 kernel (r8b_fused2.cu): persistent CTAs, one tile per half-CTA
    int n_ch;                // channels of this launch (work units = n_ch * n_tiles)
    int glog;                // log2 of the phase groups a warp covers per instruction (lanes = 32>>glog cycles x 1<<glog groups)
    int flags;               // bit 0: ping-pong token around the interpolation, bit 1: bulk-copy input tiles
    const double2* tw_tab;   // 512 entries: tw2t[q*16+r] = W_256^(r q), then tw1t[q*16+r] = W_M^(r q)
    int mbu;                 // tensor-path interpolation: blocks of 8 stepping cycles per work unit (2, 4, 6; 0 = 6)
    int n_tab, tab_off;      // the call's tile table in shared memory (r8b_fused2_core.cuh, TileEntry): entries for tile
                             // indices [0, n_tab) at byte offset tab_off; set by launch_up2_frac2
    int up;                  // BlockConvolver up-factor of the fused pair: 2 (default, also when 0) or 1
    int ylen;                // doubles of the tile's stream between the two stages held in shared memory (2*FM for up 2, FM for up 1)
    const double2* cd_tab;   // up == 2, phase C fused into the first inverse pass: [q3 < 16][g < 256] spectrum at slot 16 g + q3,
                             // then [g < 256] W_M^((g >> 4) + 16 (g & 15))
    const double2* cs_tab;   // up == 2, or nullptr: the same spectrum in its symmetric half-size form (r8b_fused2_core.cuh,
                             // cs_entry), kept in shared memory; set per plan where it fits beside the bank (fused2_cs_fits)
    const double2* c_tab;    // up == 1: phase C operands in the order the threads consume them: [u < 4][item < 3][ht < 256] --
                             // W_M^k, H[k]/2, H[N-k]/2 for k = c_freq(ht, u) -- then 3 entries for k = N/2 (v1 kernel: its own table)
};
// Template arguments of a fused-kernel launch, recorded on the host (r8bgpu_batch_last_variant):
// k_up2_frac2<ir, pad, glog, tc, up, copy, poly, cs, lin> with the call's mbu, or k_up2_frac<mode, ir, pad, bank>.
struct FusedVariant {
    int kernel = 0; // 0: none launched yet, 1: k_up2_frac, 2: k_up2_frac2
    int ir = 0, pad = 0, glog = 0, tc = 0, up = 0, copy = 0, poly = 0, cs = 0, lin = 0, mbu = 0;
    int mode = 0, bank = 0;
    // mode 1 (order-2 bank): the call's tiles and staged bank rows (FusedParams n_tiles, span, poly_dir, poly_rows_cap,
    // poly_row_stride, poly_chunks, poly_n)
    int tiles = 0, span = 0, dir = 0, rows = 0, stride = 0, chunks = 0, n = 0;
};

int fused_smem_bytes(int bank_doubles_in_smem);
int fused_max_span(int lg, int yl, int yr);
int fused_stage_doubles();
int fused_fixed_doubles();
int fused_poly_queue_bytes();
// dynamic shared memory of an order-2 launch of k_up2_frac: tile buffers and twiddles, then (poly_dir != 0) the staged
// rows and the deferred-output queue
int fused_poly_smem_bytes(int poly_dir, int poly_rows_cap, int poly_row_stride);
// variant: if not null, receives the instantiation launched (left as it was when the call has no tiles)
void launch_up2_frac(const FusedParams& p, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st,
                     FusedVariant* variant = nullptr);
// Calibration: best-of-3 TFLOP/s of a register-resident DFMA stream (16 independent chains per thread, 32 warps per
// SM) on the current device -- the fp64 ceiling the bench reports next to the HBM roofline.  < 0 on error.
double measure_dfma_tflops();

constexpr int kFused2SmemMax = 227 * 1024 - 1024; // dynamic part; the kernel's static shared memory is < 1 KB
// dynamic shared memory of k_up2_frac2: tile buffers, twiddles, the call's bank, the symmetric spectrum table (cs), the
// store staging area (r8b_hosttab.cpp)
int fused2_smem_bytes(int bank_doubles, bool cs, bool staged);
int fused2_stage_off(int bank_doubles, bool cs);
void launch_up2_frac2(const FusedParams& p, const SrcView& src, const DstView& dst, int n_sm, cudaStream_t st,
                      FusedVariant* variant = nullptr);

int blockconv_smem_bytes(int fft_log2, int up);
cudaError_t blockconv_configure(); // opt-in shared memory attributes; call once per device

void launch_blockconv(const BlockConvParams& p, const SrcView& src, const DstView& dst, int n_ch,
                      cudaStream_t st, const RaggedRec* rr = nullptr);

// Large-tile overlap-save (r8b_bclarge.cuh): a 1x BlockConvolver (also 2x and 3x on the zero-stuffed view) whose tiles of
// M = 16384 .. 65536 points are transformed as R0 = M / 4096 sub-blocks of 4096 points in shared memory, with the
// outermost radix-R0 pass through an HBM scratch buffer.
struct BcLargeParams {
    BlockConvParams bc;    // tile geometry as k_blockconv; fft_log2 14..16, spec in large slot order, tw = 4096-point twiddles
    const double2* tw_m;   // W_M^k = exp(-2 pi i k / M), k < M (device)
    double2* scratch;      // [channels of one group][tile pairs][M] (device)
    int group_ch;          // channels per launch group (the scratch holds group_ch * pairs_cap tile pairs)
};
// Runs the three kernels once per channel group; returns the number of kernel launches.
int launch_blockconv_large(const BcLargeParams& p, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st,
                           const RaggedRec* rr = nullptr);
// Fractional-delay interpolation (k_frac): one CTA computes `tile` consecutive outputs of one channel from the input
// window it stages in FRAC_CAP doubles of shared memory.  Kept small on purpose: the filter bank is read through L1 (one
// row per lane), and shared memory carved out for the window is L1 capacity lost to the bank.
constexpr int FRAC_CAP = 1536; // 12 KB
// The most window samples a tile of `tile` outputs at in_per_out input samples per output can stage: the integer input
// positions of its first and last outputs are at most floor((tile - 1) * in_per_out) + 1 apart (+ 1 more for the
// rounding of the order-2 position expression), and each output reads flen samples from its position on.
inline int frac_window(int tile, double in_per_out, int flen)
{
    return (int) std::floor((double) (tile - 1) * in_per_out) + 2 + flen;
}
// Default tile: the largest power of two up to 1024 whose window estimate fits FRAC_CAP, down to one output per CTA (whose
// window is flen samples whatever the ratio).
inline int frac_tile(double in_per_out, int flen)
{
    int tile = 1024;
    while (tile > 1 && (double) tile * in_per_out + flen + 4 > (double) FRAC_CAP) tile >>= 1;
    return tile;
}
// tile: outputs per CTA, whose frac_window must fit FRAC_CAP (the kernel traps otherwise)
void launch_frac_whole(const FracParams& p, int tile, const SrcView& src, const DstView& dst, int n_ch,
                       cudaStream_t st, const RaggedRec* rr = nullptr);
void launch_frac_poly(const FracParams& p, int tile, const SrcView& src, const DstView& dst, int n_ch,
                      cudaStream_t st, const RaggedRec* rr = nullptr);
void launch_hbup(const HbParams& p, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st,
                 const RaggedRec* rr = nullptr);
void launch_hbdown(const HbParams& p, const SrcView& src, const DstView& dst, int n_ch, cudaStream_t st,
                   const RaggedRec* rr = nullptr);
// copy cur[n0..n1) into the ring (history for later calls)
void launch_save_tail(const double* cur, long long cur_stride, long long cur_base, long long n0,
                      long long n1, double* ring, long long ring_stride, long long ring_mask, int n_ch,
                      cudaStream_t st, int fmt = 0, double scale = 1.0);
// ragged form: channel c copies cur[rr[c].m0 .. rr[c].m1) (absolute indices, cur[0] = rr[c].cur_base); n = the largest count
void launch_save_tail_ragged(const double* cur, long long cur_stride, long long n, double* ring, long long ring_stride,
                             long long ring_mask, int n_ch, cudaStream_t st, const RaggedRec* rr);

// Caller-side sample formats (r8b_format.cu); values match r8bgpu_sample_format in include/r8bgpu.h.
__host__ __device__ int format_bytes(int fmt); // bytes per element; 0: unknown format
// The element of a caller-side buffer: strides count elements, lengths count samples.  Every format holds one sample per
// element except DSD, whose byte holds 8.
struct FormatElem {
    int bytes;   // per element; 0: unknown format
    int samples; // per element
    size_t elems(long long n) const { return (size_t) (n / samples); } // elements holding n samples (a multiple of `samples`)
    size_t span(long long n) const { return elems(n) * (size_t) bytes; } // their bytes
};
FormatElem format_elem(int fmt);
// raw (any format; planar: channel c at c*raw_stride, interleaved: frame f at f*raw_stride) <-> planar fp64.
// Ragged form (rr != nullptr): n is the largest extent and channel c converts only its own -- rr[c].m1 - rr[c].cur_base
// samples into fp64 (the history record of a ragged call), rr[c].e1 - rr[c].e0 out of it (the last stage's record).
bool launch_to_f64(int fmt, const void* raw, bool interleaved, size_t raw_stride, double* f64, size_t f64_stride,
                   int n, int n_ch, double scale, cudaStream_t st, const RaggedRec* rr = nullptr);
bool launch_from_f64(int fmt, void* raw, bool interleaved, size_t raw_stride, const double* f64, size_t f64_stride,
                     int n, int n_ch, double scale, cudaStream_t st, const RaggedRec* rr = nullptr);
// Mapped form (a mixed batch): channel c's fp64 row is rec[c].row, wherever it lives, and it converts rec[c].n samples;
// n is the largest extent.  The raw side is as above.
struct MapRec {
    double* row;
    long long n;
};
bool launch_to_f64_mapped(int fmt, const void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                          double scale, cudaStream_t st);
bool launch_from_f64_mapped(int fmt, void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                            double scale, cudaStream_t st);
// Dithered integer output (r8b_dither.cuh, k_dither_shape): channel c's fp64 outputs of the call are row[0 .. n), the first
// being output n0 since its clear; n = 0 leaves the channel alone.  cfg: the channels' settings (r8bgpu_dither, whose
// layout this mirrors); err: [n_ch][16] error history, the channel's m-th dithered output's error at slot m & 15.
// shaped: the launch converts the channels with taps, each walking its frames in one pass; else the flat ones, with the
// frames split over CTAs.  fmt: S16, S24 or S32.
struct DitherRec {
    const double* row;
    long long n, n0;
    long long m0; // the channel's dithered outputs before this call: the history ring is indexed by that count
};
struct DitherCfg {
    int kind;
    unsigned long long seed;
    int n_taps;
    double taps[16];
};
// A batch's tables as one device struct, for the stores of the fused kernel (flat TPDF only).
struct DitherCall {
    const DitherCfg* cfg;
    const DitherRec* rec;
    double* err;
};
bool launch_dither(int fmt, void* raw, bool interleaved, size_t raw_stride, const DitherRec* rec, const DitherCfg* cfg, double* err,
                   int n, int n_ch, double scale, bool shaped, cudaStream_t st);

// Moving streams (r8b_state.cu): one segment of a channel's state blob -- the window [a0, a0 + len) of one power-of-two
// ring row (a stage input, or the 16-slot dither history with a0 = 0), stored as len fp64 words from `blob` on.
struct StateSeg {
    double* ring;            // the ring row (pack: read; unpack: written whole)
    double* blob;            // the window's first word in the blob
    unsigned long long* sum; // checksum accumulator (pack: the blob's checksum word; unpack check: the blob's slot)
    long long mask;          // ring capacity - 1
    long long a0, len;       // absolute index of the window's first sample, and its length
    long long lo;            // pack: samples below lo are stored as 0 (negative indices; ones the ring does not hold)
    long long word0;         // index of blob[0] among the blob's 64-bit words (the checksum weighs each word by it)
};
// The checksum term of word w at index i: SplitMix64's finaliser of w ^ (i * golden); a blob's checksum is the sum of
// the terms of all its words except the checksum word itself (mod 2^64), so segments add up in any order.
__host__ __device__ inline unsigned long long state_word_term(unsigned long long w, unsigned long long i)
{
    unsigned long long z = w ^ (i * 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
// k_state_pack: every segment's window into the blob, adding its terms to *sum.
void launch_state_pack(const StateSeg* segs, int n_segs, long long max_len, cudaStream_t st);
// k_state_unpack: check = true adds the terms of every window to *sum and writes nothing; check = false writes each
// ring row whole (mask + 1 slots): the window's values inside it, zeros elsewhere.
void launch_state_unpack(const StateSeg* segs, int n_segs, long long max_span, bool check, cudaStream_t st);

// Long clips (r8b_oneshot.cu): one record per lane and call.  Gather: samples [pos, pos + n) of the lane's clip (raw: its
// first element; interleaved frames are `stride` elements apart) widened into row[0 .. n).  Scatter: row[0 .. n) (nullptr:
// zeros) narrowed to samples [pos, pos + n) of the clip; with dither set, integer formats take the flat TPDF of output
// n0 + f of the clip (r8b_dither.cuh).
struct OneshotRec {
    const unsigned char* raw;
    double* row;
    long long pos, n, n0;
    unsigned long long seed;
    int dither;
};
bool launch_oneshot_gather(int fmt, bool interleaved, size_t stride, double scale, const OneshotRec* rec, long long max_n,
                           int n_lanes, cudaStream_t st);
bool launch_oneshot_scatter(int fmt, bool interleaved, size_t stride, double scale, const OneshotRec* rec, long long max_n,
                            int n_lanes, cudaStream_t st);

// Gradients through whole clips (r8b_adjoint.cu).  Streams are planar fp64 rows, clip r at r * stride, addressed by absolute
// sample index: the g row holds the gradient of a stage's output samples [g0, ng) (the kernels read nothing else), the x
// row receives the gradient of its input samples [x0, nx); element 0 of each row is sample g0 or x0.  A block-exact stage
// runs the blocks [b0, nb), block b's contribution at (b - b0) in the row.  Whole clips have every origin 0; crops of
// clips (r8bgpu_batch_oneshot_crops_adjoint) a window.  An order-2 interpolator's outputs run on the twin's per-call
// timing records, sorted by e0 and covering [g0, ng).
struct AdjPolyRec {
    long long e0, p0;
    double in_pos_shift, fpos0, ssr, dsr;
    int in_counter0, in_pos_int0;
};
struct AdjClip {
    long long ng, nx;
    long long nb;          // block-exact BlockConv: one past the last block
    int rec0, nrec;        // order-2 interpolator: the clip's records
    long long g0, x0, b0;  // row origins (see above)
};
struct AdjParams {
    const double* g;
    long long g_stride;
    double* x;
    long long x_stride;
    const AdjClip* clip;   // [n_clips] (device)
    // BlockConv: taps h[-L..L] (device, at h[0 .. 2L]), up U, down D
    const double* h;
    int L, U, D;
    // block-exact: blocks of il tile-stream samples, window of M from b * il - prev; kappa / u: [M] (device)
    const double* kappa;
    const double* u;
    double nyq;
    int M, il, prev;
    double* contrib;       // [n_clips][c_stride]: [block][M]
    long long c_stride;
    // interpolators
    const double* bank;
    int flen, fll, in_step, out_step, fracs;
    const AdjPolyRec* rec;
};
void launch_bc_adj(const AdjParams& p, long long max_nx, int n_clips, cudaStream_t st);
void launch_bcx_adj(const AdjParams& p, long long max_nb, long long max_nx, int n_clips, cudaStream_t st);
void launch_frac_adj(const AdjParams& p, bool poly, long long max_nx, int n_clips, cudaStream_t st);
// The input gradient of crops (k_crop_accum): clip c's samples [lo, hi) are the sums, in ascending crop order, of the rows
// of its crops whose windows [x0, x1) cover them (0 where none does), stored as F64 or F32 at the caller's row or column.
struct CropAccRow {
    long long x0, x1;      // the crop's input window
    long long row;         // its scratch row
};
struct CropAccClip {
    long long lo, hi;      // the hull of its crops' windows
    int k0, nk;            // its crops: rows[k0 .. k0 + nk), ascending crop index
    long long out;         // its row (planar) or column (interleaved) of the caller's buffer
};
struct CropAccParams {
    const double* x;
    long long x_stride;
    const CropAccRow* rows;
    const CropAccClip* clips;
    void* out;
    int fmt;               // FMT_F64 or FMT_F32
    int interleaved;
    long long out_stride;  // elements
};
void launch_crop_accum(const CropAccParams& p, long long max_hull, int n_clips, cudaStream_t st);

} // namespace r8bgpu

/* r8bgpu.h -- C-ABI of the H100-native sample-rate-conversion engine (libr8bgpu.so).
 *
 * Drop-in boundary for the r8b::CDSPResampler::process() path.  Plain C: opaque handles,
 * doubles, ints and raw pointers only -- no C++ or torch types cross this boundary.
 *
 * What each entry point replaces in the reference (file:line into avaneev/r8brain-free-src):
 *
 *   r8bgpu_plan_create            CDSPResampler::CDSPResampler()                CDSPResampler.h:117-394
 *                                 (and r8b_create()                              DLL/r8bsrc.cpp:64-88)
 *   r8bgpu_plan_max_out_len       CDSPResampler::getMaxOutLen()                 CDSPResampler.h:502-505
 *   r8bgpu_plan_in_len_before_out_pos   ::getInLenBeforeOutPos()                CDSPResampler.h:406-419
 *                                 (and r8b_inlen()                               DLL/r8bsrc.cpp:95-98)
 *   r8bgpu_plan_input_required_for_output  ::getInputRequiredForOutput()        CDSPResampler.h:476-484
 *   r8bgpu_plan_latency_frac      ::getLatencyFrac()                            CDSPResampler.h:491-494
 *   r8bgpu_batch_create           N x "new CDSPResampler24(...)", one object per channel
 *                                                                                example.cpp:30-41
 *   r8bgpu_batch_clear            CDSPResampler::clear() on every channel       CDSPResampler.h:521-529
 *                                 (and r8b_clear()                               DLL/r8bsrc.cpp:99-100)
 *   r8bgpu_batch_process          the per-channel loop "Resamps[i]->process(in[i], l, op)"
 *                                                                                example.cpp:61-67,
 *                                                                                CDSPResampler.h:559-575
 *                                 (and r8b_process()                             DLL/r8bsrc.cpp:101-105)
 *   r8bgpu_batch_process_fmt / _host_fmt   same, plus the sample conversion loops of
 *                                 oneshot<Tin,Tout>()                            CDSPResampler.h:592-651
 *   r8bgpu_batch_process_host     same, with host buffers (H2D + kernels + D2H); this is what the
 *                                 single-object r8b::CDSPResampler::process() shim in
 *                                 include/r8b/CDSPResampler.h calls.
 *   r8bgpu_batch_flush / _flush_host   the silence-feeding tail of oneshot(), then clear(), per channel
 *                                                                                CDSPResampler.h:592-651
 *
 * Conventions
 *   - Audio is planar: channel c's samples start at base + c*stride (stride in doubles).
 *   - In r8bgpu_batch_process and its typed / host forms every channel of a batch receives the
 *     same number of input samples `l` per call and therefore produces the same number of output
 *     samples, which is the return value.  Independent streams, each with its own block lengths
 *     and its own clear(), use r8bgpu_batch_process_ragged / _host_ragged and
 *     r8bgpu_batch_clear_channels (see "independent streams" below).
 *   - The reference has no error channel (R8BASSERT compiles out, r8bconf.h:20-29).  Here a
 *     negative return value / NULL handle signals failure; r8bgpu_last_error() (thread-local)
 *     says why.  There is NO CPU fallback: without a usable CUDA device every batch call fails.
 *   - A batch is bound to one CUDA device and one stream; calls on one batch must be serialised
 *     by the caller (same rule as one reference object = one thread at a time, README.md:52-55).
 *     Plans are immutable and may be shared.
 */
#ifndef R8BGPU_H_INCLUDED
#define R8BGPU_H_INCLUDED

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define R8BGPU_API __declspec(dllexport)
#else
#define R8BGPU_API __attribute__((visibility("default")))
#endif

typedef struct r8bgpu_plan r8bgpu_plan;
typedef struct r8bgpu_batch r8bgpu_batch;

/* Stage kinds reported by r8bgpu_plan_stage_info(). */
enum {
    R8BGPU_STAGE_BLOCKCONV = 0,  /* CDSPBlockConvolver  */
    R8BGPU_STAGE_FRAC_WHOLE = 1, /* CDSPFracInterpolator, whole-number stepping */
    R8BGPU_STAGE_FRAC_POLY = 2,  /* CDSPFracInterpolator, 2nd-order interpolated bank */
    R8BGPU_STAGE_HBUP = 3,       /* CDSPHBUpsampler */
    R8BGPU_STAGE_HBDOWN = 4      /* CDSPHBDownsampler */
};

typedef struct r8bgpu_stage_info {
    int kind;
    int up, down;          /* BLOCKCONV */
    int kernel_len;        /* BLOCKCONV: taps; FRAC: taps per filter; HB: one-sided taps */
    int latency;           /* BLOCKCONV: reference Latency (InputLen + L) */
    int ref_input_len;     /* BLOCKCONV: reference InputLen */
    int block_len_bits;    /* BLOCKCONV: reference BlockLenBits */
    int fracs;             /* FRAC: filter-bank fractions */
    int in_step, out_step; /* FRAC_WHOLE */
    int order;             /* FRAC: 0 or 2 */
    int max_out_len;       /* reference getMaxOutLen() chain value after this stage */
    double atten;          /* FRAC/HB: attenuation of the selected table row */
    int data_len;          /* doubles r8bgpu_plan_stage_data() provides */
} r8bgpu_stage_info;

R8BGPU_API const char* r8bgpu_last_error(void);
R8BGPU_API const char* r8bgpu_version(void);

/* ---- plan (host only; needs no GPU) ----------------------------------------------------- */

/* phase: 0 = fprLinearPhase (the only one implemented).  extfft / fasttiming carry the
 * reference's compile-time R8B_EXTFFT / R8B_FASTTIMING (r8bconf.h:132,146), which change the
 * emission timing / interpolation timing of the chain.
 * Buffer lengths: MaxInLen and every stage's max_out_len (the getMaxOutLen() chain, computed here in 64 bits) must not
 * exceed R8BGPU_MAX_LEN, or the plan is refused with a message naming the stage and its length (the reference computes
 * the chain in int and wraps).  Per-call counts are ints, so this bounds what one call can return.  The limit keeps
 * 2^16 below INT_MAX so that the kernels' 32-bit per-call grid and index arithmetic (n + 255, block * 256 + thread)
 * cannot overflow.  Sample positions within a stream are 64-bit and unbounded by it.  The same limit applies to
 * r8bgpu_plan_create_trim and r8bgpu_plan_create_stage. */
#define R8BGPU_MAX_LEN 2147418112 /* 2^31 - 2^16 */
R8BGPU_API r8bgpu_plan* r8bgpu_plan_create(double src_rate, double dst_rate, int max_in_len,
                                           double trans_band, double atten, int phase, int extfft,
                                           int fasttiming);
/* Test hook: a one-stage chain (see r8b_plan.h Plan::build_single). */
R8BGPU_API r8bgpu_plan* r8bgpu_plan_create_stage(int kind, const double* params, int n_params,
                                                 int max_in_len, int extfft);
R8BGPU_API void r8bgpu_plan_destroy(r8bgpu_plan* plan);
R8BGPU_API int r8bgpu_plan_max_out_len(const r8bgpu_plan* plan);
R8BGPU_API int r8bgpu_plan_in_len_before_out_pos(const r8bgpu_plan* plan, int req_out_pos);
R8BGPU_API int r8bgpu_plan_input_required_for_output(const r8bgpu_plan* plan, int req_out_samples);
R8BGPU_API double r8bgpu_plan_latency_frac(const r8bgpu_plan* plan);
R8BGPU_API int r8bgpu_plan_is_passthrough(const r8bgpu_plan* plan);
R8BGPU_API int r8bgpu_plan_stage_count(const r8bgpu_plan* plan);
R8BGPU_API int r8bgpu_plan_stage_info(const r8bgpu_plan* plan, int stage, r8bgpu_stage_info* info);
/* BLOCKCONV: time-domain taps h[-L..L]; FRAC: bank [(fracs+1)][taps][order+1]; HB: taps. */
R8BGPU_API int r8bgpu_plan_stage_data(const r8bgpu_plan* plan, int stage, double* out, int cap);
R8BGPU_API int r8bgpu_plan_describe(const r8bgpu_plan* plan, char* buf, int cap);
/* Dry-run of the integer scheduler: counts[i] = what process() would return for lens[i]. */
R8BGPU_API int r8bgpu_plan_simulate(const r8bgpu_plan* plan, const int* lens, int n_calls, int* counts);
/* Dry-run of a batch's per-channel schedules over n_calls ragged calls: lens and counts are [n_calls][n_channels];
 * clear (NULL: never) is [n_calls][n_channels], non-zero = r8bgpu_batch_clear_channels() on that channel just before
 * call i.  groups[i] (may be NULL) = distinct channel schedules after call i (1: the channels run in lock-step). */
R8BGPU_API int r8bgpu_plan_simulate_ragged(const r8bgpu_plan* plan, int n_channels, int n_calls, const int* lens,
                                           const int* clear, int* counts, int* groups);

/* How a batch of this plan, created now, would run a BlockConvolver stage and the interpolator behind it on its
 * lock-step calls: the decisions r8bgpu_batch_create makes, on the host, under the same R8BGPU_* settings
 * (R8BGPU_F2_FLAGS, R8BGPU_IR, R8BGPU_FUSED_V1, R8BGPU_NO_FUSION, R8BGPU_POLY_V2).  `stage` is the BlockConvolver's
 * index; another stage kind is refused.  Ragged and mixed calls run the unfused chain whatever this says. */
enum {
    R8BGPU_FUSED_NONE = 0,        /* the stage runs on its own kernel, unfused */
    R8BGPU_FUSED_F2_TC = 1,       /* k_up2_frac2, whole-stepping interpolation on the fp64 tensor path */
    R8BGPU_FUSED_F2_FMA = 2,      /* k_up2_frac2, whole-stepping interpolation in FMA loops */
    R8BGPU_FUSED_V1_SMEM = 3,     /* k_up2_frac (whole stepping), grouped bank in shared memory */
    R8BGPU_FUSED_V1_GLOBAL = 4,   /* k_up2_frac (whole stepping), grouped bank read from global memory */
    R8BGPU_FUSED_F2_COPY = 5,     /* k_up2_frac2 runs a 2x BlockConvolver alone (no interpolator fused) */
    R8BGPU_FUSED_ORDER2 = 6       /* fused with an order-2 interpolator (k_up2_frac mode 1, or k_up2_frac2<POLY>) */
};
typedef struct r8bgpu_fused_info {
    int kernel;               /* R8BGPU_FUSED_* */
    int up;                   /* up-factor of the fused BlockConvolver (1 or 2); 0 when nothing is fused */
    int copy;                 /* kernel == R8BGPU_FUSED_F2_COPY */
    int in_step, out_step;    /* the whole-stepping interpolator behind the stage (0 when there is none) */
    int tc_n_groups, tc_smaxp; /* its bank for the tensor path: ceil(out_step / 8) groups of 8 phases, padded window */
    int ir, fma_n_groups, fma_smaxp; /* its bank for the FMA loops: ir (8 or 10) phases per group */
    int pad, ysh;             /* the padded y layout of the tile (pad = ysh != 31) */
    int tc_fits, fma_fits;    /* k_up2_frac2 can hold that bank (shared memory, at most 192 groups) */
    int cs;                   /* the symmetric spectrum table is kept beside the bank (up 2 on k_up2_frac2) */
    int bank_in_smem;         /* k_up2_frac: the bank it would load fits its shared memory */
} r8bgpu_fused_info;
R8BGPU_API int r8bgpu_plan_fused_info(const r8bgpu_plan* plan, int stage, r8bgpu_fused_info* info);

/* How a batch of this plan, created now, would run half-band stage `stage` on its lock-step calls: alone, or in a
 * cascade kernel that runs up to 6 consecutive half-band stages of one direction with every intermediate rate in
 * shared memory, and that cascade's tile plan.  The decisions r8bgpu_batch_create makes, on the host, under the same
 * R8BGPU_* settings (R8BGPU_NO_FUSION, R8BGPU_NO_HB_CASCADE, R8BGPU_HB_NO_LAST2, R8BGPU_HB_SMEM_DOUBLES,
 * R8BGPU_HBD_SMEM_DOUBLES).  A stage that is not a half-band stage is refused.  For a stage inside a cascade
 * (kind R8BGPU_HB_INSIDE) only `kind` and `first` are set; ask `first` for the rest.  Ragged and mixed calls run one
 * kernel per stage whatever this says. */
enum {
    R8BGPU_HB_SINGLE = 0,         /* k_hbup or k_hbdown: the stage on its own kernel */
    R8BGPU_HB_UP_CASCADE = 1,     /* k_hbup_cascade, starting at this stage */
    R8BGPU_HB_DOWN_CASCADE = 2,   /* k_hbdown_cascade, starting at this stage */
    R8BGPU_HB_INSIDE = 3          /* inside the cascade that starts at stage `first` */
};
typedef struct r8bgpu_hb_info {
    int kind;                 /* R8BGPU_HB_* */
    int first;                /* the stage the kernel that runs this one starts at */
    int n_stages;             /* plan stages the kernel covers (1: single) */
    int ntaps[6];             /* taps of each of them, in chain order */
    int fuse_last2;           /* up cascade: its last two stages run as one pass (no buffer for the stream between) */
    int n_buffers;            /* shared-memory stream buffers: up, n_stages - fuse_last2; down, n_stages */
    int w;                    /* tile width: up, input samples of the cascade; down, outputs of its last stage */
    int smem_bytes;           /* dynamic shared memory of one CTA */
    int lo_off[7], hi_off[7]; /* up: stream k of a tile spans [2^k A - lo_off[k], 2^k (A + w) + hi_off[k]) */
    int back[7];              /* down: stream s reaches back[s] samples past 2^(n-s) m for each final output m */
    int writes_ring;          /* the kernel's output is the next stage's ring, not the call's output */
} r8bgpu_hb_info;
R8BGPU_API int r8bgpu_plan_cascade_info(const r8bgpu_plan* plan, int stage, r8bgpu_hb_info* info);

/* How a batch of this plan with n_channels channels, created now, would run BlockConvolver stage `stage` on its
 * lock-step calls: the kernel and its tile.  The decisions r8bgpu_batch_create makes, on the host, under the same
 * R8BGPU_* settings (R8BGPU_FFT_LOG2, R8BGPU_NO_FUSION, R8BGPU_FUSED_V1, R8BGPU_BCL_SCRATCH_MB and those of
 * r8bgpu_plan_fused_info).  Another stage kind, or a stage batch_create would refuse, is refused.  Ragged calls run a
 * fused or copy stage on k_blockconv with M = 4096 (fft_log2 12, as reported) and otherwise the same tile. */
enum {
    R8BGPU_BC_FUSED = 0,          /* fused with the interpolator behind it (r8bgpu_plan_fused_info) */
    R8BGPU_BC_F2_COPY = 1,        /* k_up2_frac2 runs the 2x stage alone */
    R8BGPU_BC_BLOCKCONV = 2,      /* k_blockconv<M, UP> */
    R8BGPU_BC_LARGE = 3           /* k_bcl_gather<R0> + k_bcl_conv + k_bcl_scatter<R0>, per group of channels */
};
typedef struct r8bgpu_blockconv_info {
    int kernel;               /* R8BGPU_BC_* */
    int fft_log2;             /* log2 of the tile length M */
    int up;                   /* UP of k_blockconv: 2 (polyphase 2x) or 1; 1 on the large path */
    int src_up;               /* > 1: tiles are windows of the source zero-stuffed by this factor (3x; 2x on the large path) */
    int down;                 /* every down-th output of the tile operator is kept */
    int block_exact;          /* tiles are the reference's own blocks (power-of-two decimation) */
    int trunc;                /* block_exact: down, whose Nyquist value replaces bin nyq_bin; else 0 */
    int nyq_bin;              /* M / (2 trunc) when trunc > 0, else 0 */
    int lg;                   /* half support of the filter in tile samples: outputs are valid at [lg, M - lg) */
    int adv;                  /* tile advance: the reference's input block when block_exact, else at most M - 2 lg */
    int smem_bytes;           /* dynamic shared memory of one CTA (k_blockconv, or k_bcl_conv on the large path) */
    int r0;                   /* large: M / 4096 sub-blocks */
    int scratch_tiles;        /* large: tiles of one channel's largest call the scratch holds (even) */
    long long scratch_bytes_per_ch; /* large: scratch_tiles / 2 * M * 16 */
    int group_ch;             /* large: channels per launch group of n_channels (R8BGPU_BCL_SCRATCH_MB, default 256) */
} r8bgpu_blockconv_info;
R8BGPU_API int r8bgpu_plan_blockconv_info(const r8bgpu_plan* plan, int stage, int n_channels, r8bgpu_blockconv_info* info);

/* How a batch of this plan, created now, would run interpolator stage `stage`: fused into the BlockConvolver kernel in
 * front of it, or on k_frac, one CTA per `tile` consecutive outputs of a channel that stages its input window in
 * frac_cap doubles of shared memory.  The tile is the largest power of two up to 1024 whose window fits (down to 1), or
 * R8BGPU_FRAC_TILE where that fits.  Lock-step calls size the tile from the stage's ratio (on a trim plan, from the
 * batch's common factor; reported at factor 1); ragged calls, which run every stage on k_frac, from the most input per
 * output any channel can read (a trim plan's factor 1 - max_trim).  window: the most samples a tile can stage. */
enum {
    R8BGPU_FRAC_FUSED = 0,        /* lock-step calls run the stage inside the BlockConvolver's kernel */
    R8BGPU_FRAC_WHOLE = 1,        /* k_frac<false>: whole-number stepping */
    R8BGPU_FRAC_POLY = 2          /* k_frac<true>: the order-2 bank */
};
typedef struct r8bgpu_frac_info {
    int kernel;               /* R8BGPU_FRAC_* */
    int flen, fll, fracs;     /* filter length, taps left of the position, order-2 bank rows (0 for whole stepping) */
    int tile, window;         /* lock-step calls */
    int tile_ragged, window_ragged; /* ragged calls */
    int frac_cap;             /* doubles of the staged window */
} r8bgpu_frac_info;
R8BGPU_API int r8bgpu_plan_frac_info(const r8bgpu_plan* plan, int stage, r8bgpu_frac_info* info);

/* How a lock-step call would run the fused pair of BlockConvolver stage `stage` and the order-2 interpolator behind it
 * (r8bgpu_plan_fused_info kernel R8BGPU_FUSED_ORDER2): its kernel, tiles and the run of bank rows k_up2_frac stages in
 * shared memory.  These are decided per call, from the call's rates and its span of stream positions between the two
 * stages; r8bgpu_batch_last_variant names the same fields after each such call on k_up2_frac.  trim_factor: the
 * batch's common factor on a trim plan (r8bgpu_batch_set_trim; 1 elsewhere; another factor on an ordinary plan, or one
 * outside [1 - max_trim, 1 + max_trim], is refused).  span: the call's positions [p_lo, p_hi) of the 2x stream
 * (0: a full tile pair, 2 * span_max).  The same R8BGPU_* settings as the launch path: R8BGPU_POLY_V2 (read when the
 * batch is created), R8BGPU_BANK_GLOBAL and R8BGPU_POLY_SINGLE (read on every call).  A stage that is not such a pair
 * is refused.  Ragged calls run the two stages unfused whatever this says. */
typedef struct r8bgpu_order2_info {
    int poly_v2;              /* the call runs on k_up2_frac2<POLY> (nothing below but n_tiles, span and poly_n applies) */
    int n_tiles, span;        /* tiles of the call, positions each owns (k_up2_frac: tiles in pairs, one CTA per pair) */
    int span_max;             /* the most positions one tile can own */
    int poly_dir;             /* +1 / -1: bank rows ascending / descending with the output index are staged; 0: none */
    int poly_rows_cap;        /* rows the staged run may hold */
    int poly_row_stride;      /* doubles between staged rows (3 flen, + 2 unless rows already start 4 mod 8 banks apart) */
    int poly_chunks;          /* a pair's outputs are processed in this many pieces, each with its own run */
    int poly_n;               /* 1..3: four consecutive outputs per thread share their row loads (poly_block4<N>); 0: one */
    int ysh;                  /* y layout of the tile buffers: index i at i + (i >> ysh); 31 plain */
    int smem_bytes;           /* dynamic shared memory of k_up2_frac (0 on k_up2_frac2) */
    int flen, fracs;          /* the order-2 bank: taps per row, rows */
    double ratio;             /* ssr / dsr of the call: input positions per output */
} r8bgpu_order2_info;
R8BGPU_API int r8bgpu_plan_order2_info(const r8bgpu_plan* plan, int stage, double trim_factor, int span,
                                       r8bgpu_order2_info* info);

/* ---- batch (GPU) ------------------------------------------------------------------------- */

R8BGPU_API int r8bgpu_device_count(void);
/* device >= 0: that CUDA device.  R8BGPU_DEVICE_ALL (-1): every visible device -- the channels are sharded
 * contiguously, ceil(n/G) per GPU, and each shard is an ordinary single-device batch driven by its own worker thread
 * (bound to the GPU's NUMA node), stream set and PCIe link; there is no device-to-device traffic.  Such a batch takes
 * HOST buffers (r8bgpu_batch_process_host / _host_fmt); device buffers go to the shards (r8bgpu_batch_shard()).  With
 * one visible device, or one channel, this is an ordinary batch.  R8BGPU_DEVICE_CURRENT (-2): the current device.
 * Replaces the caller-side loop over per-channel objects spread over threads (example.cpp:30-67). */
#define R8BGPU_DEVICE_ALL (-1)
#define R8BGPU_DEVICE_CURRENT (-2)
R8BGPU_API r8bgpu_batch* r8bgpu_batch_create(const r8bgpu_plan* plan, int n_channels, int device);
/* Shards of a batch (1 for a single-device batch): device, channel range and NUMA node (-1: unknown / one node). */
R8BGPU_API int r8bgpu_batch_shard_count(const r8bgpu_batch* batch);
R8BGPU_API int r8bgpu_batch_shard_info(const r8bgpu_batch* batch, int shard, int* device, int* first_channel,
                                       int* n_channels, int* numa_node);
/* The single-device batch behind shard `shard` (owned by `batch`; for device-pointer calls on its GPU). */
R8BGPU_API r8bgpu_batch* r8bgpu_batch_shard(r8bgpu_batch* batch, int shard);
/* Page-locked planar host buffer [channels][samples_per_channel] of `sample_bytes`-wide samples whose rows sit on the
 * NUMA node of the GPU that owns the channel (mmap + mbind + cudaHostRegister); free with r8bgpu_host_free(). */
R8BGPU_API void* r8bgpu_batch_host_alloc(const r8bgpu_batch* batch, size_t samples_per_channel, int sample_bytes);
R8BGPU_API void r8bgpu_batch_destroy(r8bgpu_batch* batch);
R8BGPU_API int r8bgpu_batch_clear(r8bgpu_batch* batch);
R8BGPU_API int r8bgpu_batch_channels(const r8bgpu_batch* batch);
/* stream: a cudaStream_t (NULL = the legacy default stream, which is also the default). */
R8BGPU_API int r8bgpu_batch_set_stream(r8bgpu_batch* batch, void* stream);

/* Device-pointer call; asynchronous on the batch's stream.  l <= MaxInLen.  Output sample i of
 * channel c lands in d_out[c*out_ch_stride + i]; out_cap is the room per channel (use
 * r8bgpu_plan_max_out_len()).  Returns samples produced per channel, or < 0. */
R8BGPU_API int r8bgpu_batch_process(r8bgpu_batch* batch, const double* d_in, size_t in_ch_stride, int l,
                                    double* d_out, size_t out_ch_stride, int out_cap);
/* Host-pointer call: copies in, runs, copies the produced samples out, synchronises. */
R8BGPU_API int r8bgpu_batch_process_host(r8bgpu_batch* batch, const double* h_in, size_t in_ch_stride,
                                         int l, double* h_out, size_t out_ch_stride, int out_cap);
R8BGPU_API int r8bgpu_batch_sync(r8bgpu_batch* batch);

/* ---- independent streams ------------------------------------------------------------------
 * One batch channel = one reference object with its own process(ip, l, op) and clear() (README.md:52-55 of the
 * reference: one resampler object per channel or stream).  lens[c] (host array, 0..MaxInLen) is channel c's block
 * length this call; counts[c] receives the samples channel c produced, known when the call returns because the
 * schedules live on the host.  Returns 0, or < 0.  The device form is asynchronous like r8bgpu_batch_process(); the
 * host form synchronises and, on an R8BGPU_DEVICE_ALL batch, hands each shard its channel range.  Channel c's input
 * is read from in + c*in_ch_stride (lens[c] samples) and its output written to out + c*out_ch_stride.
 * After a ragged call or a per-channel clear the channels' schedules may differ: r8bgpu_batch_process /
 * _process_host then run as a ragged call with equal lengths and return the common count, or fail when the channels
 * would produce different counts; the typed-buffer calls (_fmt) need channels in lock-step, and the typed ragged
 * calls (r8bgpu_batch_process_ragged_fmt / _host_ragged_fmt, below) take typed buffers at any time.  Once every channel is in
 * the same state again (for example after r8bgpu_batch_clear), the batch runs lock-step as before.
 * R8B_FASTTIMING plans refuse ragged calls and per-channel clears of a subset. */
R8BGPU_API int r8bgpu_batch_process_ragged(r8bgpu_batch* batch, const double* d_in, size_t in_ch_stride,
                                           const int* lens, double* d_out, size_t out_ch_stride, int out_cap,
                                           int* counts);
R8BGPU_API int r8bgpu_batch_process_host_ragged(r8bgpu_batch* batch, const double* h_in, size_t in_ch_stride,
                                                const int* lens, double* h_out, size_t out_ch_stride, int out_cap,
                                                int* counts);
/* CDSPResampler::clear() (CDSPResampler.h:521-529) on channels[0..n-1] only; synchronises. */
R8BGPU_API int r8bgpu_batch_clear_channels(r8bgpu_batch* batch, const int* channels, int n);
/* Distinct channel schedules (1: the channels run in lock-step; a multi-device batch sums its shards). */
R8BGPU_API int r8bgpu_batch_channel_groups(const r8bgpu_batch* batch);

/* ---- caller-side sample formats ---------------------------------------------------------
 * What the reference's callers do on the CPU around process(): CDSPResampler::oneshot<Tin,Tout>()
 * converts "(double) ip[i]" on the way in and "(Tout) op[i]" on the way out (CDSPResampler.h:592-651),
 * and WAV front-ends de-interleave frames (bench/r8bfreesrc.cpp:106-137).  Here the narrow samples
 * cross PCIe / HBM as they are and are widened / narrowed on the device.
 *   in : x = (double) v * scale        out: v = (T) (y * scale)
 * With scale = 1 these are exactly the C++ conversions of oneshot(): widening is exact, float output
 * rounds to nearest, integer output truncates toward zero (out-of-range values, undefined in the
 * reference, saturate; NaN -> 0).  R8BGPU_S24 is packed 3-byte little-endian.
 * One-byte formats (planar or interleaved, stride in samples, the same scale):
 *   R8BGPU_U8   unsigned 8-bit PCM (WAV), silence at 128.  in: x = (double) (v - 128) * scale.  out: q + 128, q the int8
 *               value by the integer rule above with range -128..127 (or the dithered value when the channel's dither is on).
 *   R8BGPU_ULAW G.711 mu-law (RTP payload type 0).  in: x = (double) D(v) * scale.  out: E(s), s the int16 value the same
 *               call stores for R8BGPU_S16 with the same scale and the channel's dither setting.
 *   R8BGPU_ALAW G.711 A-law (RTP payload type 8), as R8BGPU_ULAW.
 * D / E are G.711 expansion to / compression from 16-bit linear in the convention of Sun's public-domain g711.c (as in
 * CPython's audioop): mu-law 0x00 -> -32124, 0x80 -> +32124, 0x7F and 0xFF -> 0; A-law 0x2A -> -32256, 0xAA -> +32256,
 * 0x55 -> -8, 0xD5 -> +8.  With scale = 1/32768 they map to about [-1, 1), like int16.  So on every path the mu-law / A-law
 * bytes of a call are the G.711 encoding of the int16 values it would write as R8BGPU_S16: dither and noise shaping act
 * in the 16-bit domain and the error history is the S16 one.  U8 is an integer format wherever the dither rules say so.
 * Silence (a passthrough plan's flush) is the encoding of 0: 128, 0xFF and 0xD5.
 * One-bit formats (DSD: SACD, DSF and DSDIFF files at 2822400 Hz and its multiples), input, and output by opt-in:
 *   R8BGPU_DSD_LSB  DSF bit order: bit 0 of each byte is the earliest sample.
 *   R8BGPU_DSD_MSB  DSDIFF (DFF) bit order: bit 7 of each byte is the earliest sample.
 *               in: bit 1 -> +scale, bit 0 -> -scale (exact).  SACD's 0 dB level is 50 % modulation; scale 0.5 is common.
 *               An element is one byte holding 8 consecutive samples of one channel, and stride counts elements (bytes):
 *               planar, sample i of channel c is in byte c*stride + i/8; interleaved (DSDIFF's byte interleave), in byte
 *               (i/8)*stride + c; the bit is i % 8 (LSB) or 7 - i % 8 (MSB).  Lengths (l, lens[c], MaxInLen) still count
 *               samples and must be multiples of 8: one DSF block group (4096 bytes per channel) is a planar buffer with
 *               stride 4096 and l = 32768.  As an output, either is refused ("DSD formats are input-only") unless the
 *               batch has DSD output on (r8bgpu_batch_set_dsd_out, "one-bit DSD output" below).
 * Values 8..15 and above R8BGPU_DSD_MSB are refused. */
typedef enum {
    R8BGPU_F64 = 0,
    R8BGPU_F32 = 1,
    R8BGPU_S16 = 2,
    R8BGPU_S24 = 3,
    R8BGPU_S32 = 4,
    R8BGPU_U8 = 5,
    R8BGPU_ULAW = 6,
    R8BGPU_ALAW = 7,
    R8BGPU_DSD_LSB = 16,
    R8BGPU_DSD_MSB = 17
} r8bgpu_sample_format;

typedef struct {
    void* data;      /* host (…_host_fmt) or device (…_fmt) memory; never written when used as input */
    int format;      /* r8bgpu_sample_format */
    int interleaved; /* 0: planar, channel c starts at c*stride; 1: frame f starts at f*stride, channel c at +c */
    size_t stride;   /* in elements of `format`: samples, or bytes of 8 samples for DSD */
    double scale;    /* see above; 1.0 for the reference's plain casts */
} r8bgpu_buffer;

/* As r8bgpu_batch_process() / r8bgpu_batch_process_host() with typed buffers.  out_cap = room per
 * channel in samples. */
R8BGPU_API int r8bgpu_batch_process_fmt(r8bgpu_batch* batch, const r8bgpu_buffer* d_in, int l,
                                        const r8bgpu_buffer* d_out, int out_cap);
R8BGPU_API int r8bgpu_batch_process_host_fmt(r8bgpu_batch* batch, const r8bgpu_buffer* h_in, int l,
                                             const r8bgpu_buffer* h_out, int out_cap);
/* Independent streams with typed buffers: r8bgpu_batch_process_ragged / _host_ragged (lens, counts, return value,
 * device / host forms, shards) combined with the conversions above; the channels need not be in lock-step.
 *   planar     : channel c reads lens[c] samples from data + c*stride and writes counts[c] samples at data + c*stride.
 *   interleaved: channel c is column c, frames [0, lens[c]) in and [0, counts[c]) out; the input buffer must hold
 *                max(lens) frames (the host form copies that many frames of every column).
 * Nothing past counts[c] is written in either layout, and the input is never written.  Plain buffers (planar
 * R8BGPU_F64, scale 1) run exactly as r8bgpu_batch_process_ragged / _host_ragged. */
R8BGPU_API int r8bgpu_batch_process_ragged_fmt(r8bgpu_batch* batch, const r8bgpu_buffer* d_in, const int* lens,
                                               const r8bgpu_buffer* d_out, int out_cap, int* counts);
R8BGPU_API int r8bgpu_batch_process_host_ragged_fmt(r8bgpu_batch* batch, const r8bgpu_buffer* h_in, const int* lens,
                                                    const r8bgpu_buffer* h_out, int out_cap, int* counts);

/* ---- end of stream ------------------------------------------------------------------------
 * The tail of CDSPResampler::oneshot() (CDSPResampler.h:592-651) per channel: after its last real input, channel
 * channels[i] is fed silence until its output since its last clear reaches targets[i], returns the samples from its
 * current output position up to that target, and is then cleared (its next call starts a fresh stream).
 *   - targets == NULL: the default target ceil(N * dst / src), N = the channel's input samples since its last clear,
 *     computed exactly on the binary values of the two rates (no rounding).  Explicit targets are absolute output
 *     counts since the last clear (see r8bgpu_batch_channel_totals).
 *   - counts[c] = max(0, target - outputs already produced) for a named channel, 0 for every other channel.  A target
 *     already reached writes nothing and still clears the channel (oneshot() with a small oplen).
 *   - Channels not named take no input, produce no output and keep their state; nothing is written in their rows /
 *     columns, and nothing past counts[c] in any.
 *   - Output rules follow r8bgpu_buffer (planar or interleaved, every format, scale); out_cap = room per channel.
 *     Passthrough plans (src == dst) write counts[c] zeros.
 *   - The silence never exists as a buffer: it is neither copied over PCIe nor built in device memory.
 *   - A refused call (bad or repeated channel index, negative target, out_cap too small, R8B_FASTTIMING plan) changes
 *     neither the schedules nor the rings.  R8B_FASTTIMING plans refuse every flush.
 * The device form is asynchronous on the batch stream (counts are known when it returns) and is refused on a
 * multi-device batch (call its shards); the host form synchronises and, on an R8BGPU_DEVICE_ALL batch, hands each shard
 * its channels once every shard has accepted the call. */
R8BGPU_API int r8bgpu_batch_flush(r8bgpu_batch* batch, const int* channels, int n, const long long* targets,
                                  const r8bgpu_buffer* d_out, int out_cap, int* counts);
R8BGPU_API int r8bgpu_batch_flush_host(r8bgpu_batch* batch, const int* channels, int n, const long long* targets,
                                       const r8bgpu_buffer* h_out, int out_cap, int* counts);
/* Each channel's input and output sample totals since its last clear (arrays of r8bgpu_batch_channels() entries). */
R8BGPU_API int r8bgpu_batch_channel_totals(const r8bgpu_batch* batch, long long* n_in, long long* n_out);
/* An upper bound of what a default-target flush returns for any channel state: size out_cap with it.  Derived from
 * per-stage lower bounds of the emitted counts (r8b_plan.cpp, flush_max_out_len); 0 for passthrough plans. */
R8BGPU_API int r8bgpu_plan_flush_max_out_len(const r8bgpu_plan* plan);
/* Dry run of one channel (no GPU): n_calls blocks of lens[i] samples, then a flush to `target` (< 0: the default
 * target).  *zeros_fed = the silence fed (the smallest length that reaches the target), *count = samples returned.
 * Constant memory; time grows with the silence fed over MaxInLen, as the flush's own planning does. */
R8BGPU_API int r8bgpu_plan_simulate_flush(const r8bgpu_plan* plan, int n_calls, const int* lens, long long target,
                                          long long* zeros_fed, int* count);

/* ---- mixed batches ------------------------------------------------------------------------
 * Independent streams at different rates in one batch: channel c runs plans[plan_of[c]], exactly as a reference object
 * constructed with that plan's parameters and fed the same blocks (README.md:52-55 of the reference: one object per
 * stream, each with its own rates).  Channels of different plans may sit in any order in the caller's buffers.
 *   - The plans must share one MaxInLen; any mix of rates, transition bands, attenuations, R8B_EXTFFT and passthrough
 *     (src == dst) plans is allowed.  Refused: R8B_FASTTIMING plans, a plan_of entry out of range, a plan without a
 *     channel, and device R8BGPU_DEVICE_ALL (one device, or R8BGPU_DEVICE_CURRENT).
 *   - Behind the handle there is one ordinary batch per plan (its part, holding that plan's channels in ascending
 *     order), and each part runs on its own stream, so small parts overlap.  Every call is planned on every part
 *     before any part runs: a refused call changes nothing.
 *   - Work per channel: r8bgpu_batch_process_ragged / _host_ragged / _ragged_fmt / _host_ragged_fmt (out_cap at least
 *     r8bgpu_batch_max_out_len()), r8bgpu_batch_clear / _clear_channels, r8bgpu_batch_flush / _flush_host (default
 *     target: each channel's own ceil(N * dst / src); out_cap as for an ordinary batch, r8bgpu_batch_flush_max_out_len()
 *     bounds a default flush), _channel_totals, _set_stream, _sync, _host_alloc.  The device forms stay asynchronous
 *     on the batch stream.  Plain fp64 buffers take the same two mapped conversions as typed ones.
 *   - Summed over the parts: _channel_groups, _kernel_launches (plus the batch's own conversion launches) and
 *     _device_bytes (plus the batch's records and host-form blocks).
 *   - Refused, because the channels produce different counts or a stage index means nothing across plans:
 *     r8bgpu_batch_process / _process_host / _process_fmt / _process_host_fmt, r8bgpu_batch_stage_kernel and
 *     r8bgpu_batch_stage_time_ms (ask the parts, r8bgpu_batch_part()). */
R8BGPU_API r8bgpu_batch* r8bgpu_batch_create_mixed(const r8bgpu_plan* const* plans, int n_plans, const int* plan_of,
                                                   int n_channels, int device);
/* Room per channel a call needs: the plan's r8bgpu_plan_max_out_len() / _flush_max_out_len(), or on a mixed batch the
 * largest of its plans' values. */
R8BGPU_API int r8bgpu_batch_max_out_len(const r8bgpu_batch* batch);
R8BGPU_API int r8bgpu_batch_flush_max_out_len(const r8bgpu_batch* batch);
/* The ordinary batch behind plans[plan_index] of a mixed batch (owned by `batch`), for introspection only:
 * r8bgpu_batch_stage_kernel, _kernel_launches, _set_timing / _stage_time_ms, _channel_groups. */
R8BGPU_API r8bgpu_batch* r8bgpu_batch_part(r8bgpu_batch* batch, int plan_index);

/* ---- per-channel rate trim ----------------------------------------------------------------
 * A live source labelled `src` Hz runs on its own clock and really delivers src * (1 +- eps) samples per second, eps of
 * some 10 to a few hundred ppm, wandering with temperature.  A receiver that keeps a fixed ratio lets its buffer drift
 * until it under- or over-runs; rebuilding the plan loses the stream's state.  Asynchronous resampling instead trims each
 * stream's ratio by a few ppm per block, driven by the caller's own control loop (which watches its buffer's fill
 * level).  The engine takes the factors; choosing them is the caller's job.
 *
 * Trim plan.  r8bgpu_plan_create_trim(src, dst, max_in_len, trans_band, atten, extfft, max_trim), 0 < max_trim <= 0.01:
 *   - the chain the reference builds for (src, dst), with one difference: its fractional interpolator is always the
 *     order-2 bank (R8BGPU_STAGE_FRAC_POLY), never whole stepping, since whole stepping cannot change its ratio without
 *     changing its filter bank.  No fasttiming argument: R8B_FASTTIMING is not offered.  Refused, each with its own
 *     message: max_trim out of range, passthrough pairs (src == dst), and chains without an interpolator (integer and
 *     power-of-two ratios); r8bgpu_plan_create_asrc (below) plans those pairs too.
 *   - max_out_len, src_history and ring sizes are those of the factor 1 + max_trim, so every factor in range fits the
 *     buffers.  r8bgpu_plan_max_out_len reports that largest-factor bound (size out_cap with it); the other r8bgpu_plan_*
 *     accessors (in_len_before_out_pos, input_required_for_output, latency_frac, stage_info, simulate) describe factor 1.
 *   - The low-pass filters stay those designed for (src, dst): exact on upsampling chains, whose filters depend on src and
 *     the attenuation only, and slightly off-design at the transition band's edge on downsampling chains.
 * Factor per channel.  r8bgpu_batch_set_trim(batch, channels, n, factors), r8bgpu_batch_trim(batch, factors):
 *   - factors[i] must lie in [1 - max_trim, 1 + max_trim]; channel channels[i] then produces about dst * f samples per src
 *     input samples.  Its interpolator runs with exactly the (ssr, dsr) doubles the planner derives on this chain for
 *     dst' = fl(dst * f): the product is rounded once, then the planner's usual stage arithmetic applies.
 *   - A new factor takes effect at the start of the channel's next call, through the reference's own re-base of the
 *     interpolator position (CDSPFracInterpolator.h:907-919: InPosShift = fpos * dsr / ssr, InCounter = InPosInt = 0)
 *     done with the new dsr, so the read position stays continuous.  Setting the same factor again does nothing: no
 *     re-base, the same bits.
 *   - Factors survive r8bgpu_batch_clear and _clear_channels: they are control-loop settings, not stream state.
 *   - Refused, changing nothing: a channel whose plan is not a trim plan, a factor out of range, a repeated channel.
 *   - Accepted on ordinary single-device batches, on mixed batches (trim plans may be parts; each channel goes to its
 *     part) and on R8BGPU_DEVICE_ALL batches (channel ranges go to the shards).  r8bgpu_batch_trim reports 1 for channels
 *     of ordinary parts.
 * Calls on a trim batch follow the rules of a diverged batch (independent streams, above): channels with equal factors
 * and equal states share one schedule group; a batch whose channels all share one factor and one state runs lock-step
 * with that factor's rates; r8bgpu_batch_process returns the common count or fails when the counts differ.
 * Flushes need explicit targets: the default ceil(N * dst / src) means nothing once the ratio has moved, so targets ==
 * NULL, r8bgpu_plan_flush_max_out_len and r8bgpu_batch_flush_max_out_len are refused on a trim plan.
 * r8bgpu_plan_simulate_trim: one channel without a GPU, through the batch's own host code.  Block i (lens[i] samples) is
 * fed after factor factors[i] has been set; counts[i] = the samples it produces.  next_pos / next_frac (may be NULL)
 * receive the interpolator's read position after call i: the integer index into its input stream of its next output,
 * and that output's fraction.
 *
 * Trim plan for any rate pair.  r8bgpu_plan_create_asrc(src, dst, max_in_len, trans_band, atten, extfft, max_trim) takes
 * the arguments of r8bgpu_plan_create_trim and follows its contract, but accepts every rate pair, src == dst included:
 * two devices "both at 48 kHz" on different crystals, or 44100 -> 88200 from a drifting source.
 *   - Where r8bgpu_plan_create_trim accepts the pair, the plan is the same: the same stages, stage data, max_out_len,
 *     state fingerprint and simulate_trim output.
 *   - Elsewhere the reference's constructor takes a shortcut that builds no interpolator (the passthrough return, the
 *     single-step ratios 1:2, 1:3, 2:3, 3:2, 3:4, whole 2^c / 3*2^c upsampling, exact 2x / 3x decimation).  This plan
 *     skips exactly those shortcuts and keeps every other decision of the constructor, so the chain is the one it builds
 *     at a rate a few ppm away: 48000 -> 48000 is a 2x BlockConvolver and an order-2 interpolator 96000 -> 48000;
 *     44100 -> 88200 interpolates at ratio 1 behind a 2x BlockConvolver; 96000 -> 48000 is a 1x BlockConvolver at 1/2
 *     and an interpolator.
 *   - The plan is never a passthrough plan (r8bgpu_plan_is_passthrough returns 0); its stage count and fingerprint keep
 *     it apart from the passthrough plan of the same rates, so a state blob of one is refused by the other.
 *   - Everything above applies: factors, re-base, (ssr, dsr) for fl(dst * f), explicit flush targets, diverged-batch
 *     calls, mixed parts, R8BGPU_DEVICE_ALL, dither, export / import. */
R8BGPU_API r8bgpu_plan* r8bgpu_plan_create_trim(double src_rate, double dst_rate, int max_in_len, double trans_band,
                                                double atten, int extfft, double max_trim);
R8BGPU_API r8bgpu_plan* r8bgpu_plan_create_asrc(double src_rate, double dst_rate, int max_in_len, double trans_band,
                                                double atten, int extfft, double max_trim);
/* 0 for an ordinary plan. */
R8BGPU_API double r8bgpu_plan_max_trim(const r8bgpu_plan* plan);
R8BGPU_API int r8bgpu_plan_simulate_trim(const r8bgpu_plan* plan, int n_calls, const int* lens, const double* factors,
                                         int* counts, long long* next_pos, double* next_frac);
R8BGPU_API int r8bgpu_batch_set_trim(r8bgpu_batch* batch, const int* channels, int n, const double* factors);
R8BGPU_API int r8bgpu_batch_trim(const r8bgpu_batch* batch, double* factors);

/* ---- dithered integer output --------------------------------------------------------------
 * The typed calls narrow to int16 / packed int24 / int32 with the reference's plain C cast (T) (y * scale), as
 * CDSPResampler::oneshot<Tin,Tout>() does (CDSPResampler.h:592-651): truncation toward zero, a bias of up to 1 LSB and
 * signal-correlated distortion on quiet material.  The reference leaves proper quantisation to its caller, between
 * process() and the cast (README.md:178 points to a PRNG for dithering); here the cast runs on the device, so the
 * dither does too.  Each channel has a setting: OFF (the default: exactly the cast) or TPDF, optionally noise-shaped by
 * caller-supplied error-feedback taps.
 *
 * Contract, per channel and integer output only (S16, S24, S32, U8, and ULAW / ALAW through their int16 value).  n = the sample's index among the channel's outputs since its last
 * clear (the count r8bgpu_batch_channel_totals reports; flush outputs count).  For output n with fp64 value y:
 *   1. v = fl(y * scale).
 *   2. z = seed + (n + 1) * 0x9E3779B97F4A7C15 (mod 2^64); SplitMix64's finaliser: z ^= z >> 30; z *= 0xBF58476D1CE4E5B9;
 *      z ^= z >> 27; z *= 0x94D049BB133111EB; z ^= z >> 31; d = (z >> 32) * 2^-32 - (z & 0xFFFFFFFF) * 2^-32, exact,
 *      triangular on (-1, 1) LSB.
 *   3. s = 0; for k = K down to 1: s = fl(s + fl(c_k * e[n-k])) (no FMA; e[j] = 0 before the first output since the
 *      clear); w = fl(v - s).
 *   4. q = rint(fl(w + d)) (half to even); e[n] = fl(q - w), from the unclipped q, so |e| <= 1.5 for any taps.
 *   5. The stored value is q saturated to the format's range.  A non-finite v stores what the cast stores (NaN -> 0,
 *      +-inf -> the limits) and sets e[n] = 0.
 * So the bytes depend on the setting, the channel's fp64 stream and n only -- not on chunking, buffer layout, batch width,
 * channel slot or kernel path.
 * Rules:
 *   - F32 / F64 outputs are never dithered.  Float-output calls, and calls while the channel is OFF, leave its error
 *     history untouched (e[n-k] above is the error of the channel's k-th most recent dithered output); n advances.
 *   - Settings survive r8bgpu_batch_clear, _clear_channels and flushes (like trim factors); the stream state (n, the
 *     error history) restarts wherever the channel is cleared.  Setting a channel again keeps its history; new taps
 *     apply from its next output.
 *   - OFF channels produce exactly the cast's bytes on every path, whatever their neighbours are set to.
 * r8bgpu_batch_set_dither(batch, channels, n, cfg): cfg[i] for channel channels[i].  Refused, changing nothing: an unknown
 * kind, n_taps outside 0..R8BGPU_DITHER_MAX_TAPS, taps with kind OFF, a non-finite tap, a channel out of range or named
 * twice.  Accepted on ordinary batches, on mixed batches (the settings stay with the batch, which owns the conversions
 * into the caller's buffer) and on R8BGPU_DEVICE_ALL batches (channel ranges go to the shards).
 * Where it runs: flat TPDF in the stores of the fused kernel's typed output (lock-step calls that narrow there);
 * otherwise the usual conversion runs and one more kernel (k_dither_shape) re-quantises the dithered channels from the
 * call's fp64 outputs.  OFF channels keep the bytes of the usual conversion.
 * r8bgpu_dither_quantize_host(cfg, fmt, scale, y, n, first_index, err_state, out): the same quantiser on the host for one
 * planar channel: y[0..n) are outputs first_index.., out receives n samples of fmt (S16, S24 packed, S32, or one byte each
 * for U8, ULAW, ALAW; with kind OFF the plain cast, encoded for ULAW / ALAW), err_state (16 doubles, zero after a clear)
 * carries the error history between calls, newest first. */
#define R8BGPU_DITHER_OFF 0
#define R8BGPU_DITHER_TPDF 1
#define R8BGPU_DITHER_MAX_TAPS 16
typedef struct r8bgpu_dither {
    int kind;                 /* R8BGPU_DITHER_OFF / _TPDF */
    unsigned long long seed;
    int n_taps;               /* 0 .. R8BGPU_DITHER_MAX_TAPS: error-feedback taps c_1 .. c_K (0: flat TPDF) */
    double taps[R8BGPU_DITHER_MAX_TAPS];
} r8bgpu_dither;
R8BGPU_API int r8bgpu_batch_set_dither(r8bgpu_batch* batch, const int* channels, int n, const r8bgpu_dither* cfg);
R8BGPU_API int r8bgpu_dither_quantize_host(const r8bgpu_dither* cfg, int fmt, double scale, const double* y, int n,
                                           long long first_index, double* err_state, void* out);

/* ---- one-bit DSD output -------------------------------------------------------------------
 * PCM to DSF / DSDIFF bytes: each channel's fp64 outputs drive a 7th-order one-bit sigma-delta modulator on the device,
 * one channel per lane (the recursion is sequential in time; channels are independent).  Opt in per batch with
 * r8bgpu_batch_set_dsd_out(batch, 1); refused, changing nothing, unless every plan of the batch (every part of a mixed
 * batch) has a DSD destination rate: 64, 128, 256 or 512 x 44100 or 48000.  Turning it on (again) zeroes every channel's
 * modulator; turning it off (0) drops the modulators, and outputs are as before.
 * The modulator, per channel and output n with fp64 value y (every operation one correctly rounded fp64 operation, no
 * FMA; state ep = e[n-1], p_1..p_7, all 0 after a clear):
 *   1. v = fl(y * scale), a non-finite v is 0, v clamped to [-0.5, 0.5] (SACD's 0 dB: 50 % modulation).
 *   2. u = fl(fl(g_1 * ep) + fl(v + p_1)).
 *   3. The bit is u >= 0 (1 = +1, 0 = -1); q = +1 or -1.
 *   4. If not |u| <= 4: ep and p_1..p_7 become 0, the channel counts one overload, and the output ends here.
 *   5. e = fl(q - u); f = fl(fl(g_1 * ep) + p_1); r_k = fl(fl(g_k * ep) + p_k) (k = 2..7); p_k = fl(r_{k+1} + fl(-a_k * f))
 *      (k = 1..6), p_7 = fl(-a_7 * f); ep = e.
 * This is the loop filter NTF - 1 = G / A in transposed direct form II, arranged so that three operations separate e[n]
 * from u[n+1].  NTF = B / A: a zero at DC and three conjugate pairs at 22050 Hz x the positive roots of the 7th Legendre
 * polynomial (at 2822400 Hz), and 7th-order Butterworth high-pass poles with max |NTF| = 1.3; g_k = b_k - a_k:
 *   g = -0.52235343612653207, 3.000835998986414, -7.1916327798335757, 9.2026607872978481, -6.631444183027881,
 *       2.5513679570436851, -0.40943457836890584
 *   a = -6.4737547313163422, 17.979709100302625, -27.769461679678152, 25.758433672213886, -14.349100916261154,
 *       4.4447402103991882, -0.59056542163109382
 * (the exact binary values: r8b_dsdmod.cuh, written by tools/dsd_ntf.py).  No dither: over 2 s of silence no in-band
 * spectral line rises above -140 dB re a 0.5 sine.  The stream's bytes are a function of the channel's fp64 outputs alone, never of chunking, buffer layout,
 * batch width, channel slot or shard.
 * While it is on:
 *   - Outputs must be R8BGPU_DSD_LSB or _MSB (planar or interleaved, the layout and stride rules of DSD input); any other
 *     output format, and the fp64-only calls (r8bgpu_batch_process, _process_host, _process_ragged, _process_host_ragged),
 *     are refused.  The calls that take DSD: _process_fmt / _process_host_fmt, _process_ragged_fmt /
 *     _process_host_ragged_fmt, _flush / _flush_host; on ordinary batches, mixed batches (the batch keeps the state) and
 *     R8BGPU_DEVICE_ALL batches (the setting and each channel range go to the shards).
 *   - Counts are whole bytes, multiples of 8 samples: a call returns floor((held + produced) / 8) * 8 bits per channel,
 *     and the up to 7 bits of an unfinished byte are held back and written first by the channel's next call.  out_cap
 *     must be at least r8bgpu_batch_max_out_len(), which reports floor((max_out_len + 7) / 8) * 8.  Lock-step calls need
 *     every channel to hold back the same number of bits (true unless ragged calls made them differ).
 *   - A flush ends each named channel on a whole byte: the modulator runs on past the resampler's tail with silence
 *     (y = 0) to the next byte boundary, and the channel restarts.  Explicit targets must be multiples of 8.
 *     r8bgpu_batch_flush_max_out_len() reports floor((flush_max_out_len + 14) / 8) * 8 (held-back bits plus the fill).
 *   - r8bgpu_batch_channel_totals still counts resampler outputs.
 *   - r8bgpu_batch_clear and _clear_channels zero the named channels' modulators and overload counts; a flush restarts
 *     the modulator (filter and held-back bits) but keeps the count, so a stream's overloads, its flush included, can be
 *     read after its flush.
 *   - r8bgpu_batch_export / _import (and the device forms) are refused: the blob (version 1) carries no modulator state.
 * r8bgpu_batch_dsd_overloads(batch, counts): each channel's overloads since its last clear / _clear_channels (or since
 * DSD output was turned on), flushes included (synchronises).  With timing on (r8bgpu_batch_set_timing), the modulator's
 * launches are timed as stage r8bgpu_plan_stage_count(plan) of r8bgpu_batch_stage_time_ms.
 * r8bgpu_dsd_modulate_host(scale, y, n, state, bits, overloads): the same modulator on the host for one channel: bits[i]
 * = 0 / 1 for y[i]; state holds 8 doubles (ep, p_1..p_7; zeros to start) carried between calls; *overloads is
 * incremented. */
R8BGPU_API int r8bgpu_batch_set_dsd_out(r8bgpu_batch* batch, int on);
R8BGPU_API int r8bgpu_batch_dsd_overloads(r8bgpu_batch* batch, long long* counts);
R8BGPU_API int r8bgpu_dsd_modulate_host(double scale, const double* y, int n, double* state, unsigned char* bits,
                                        long long* overloads);

/* ---- moving streams -----------------------------------------------------------------------
 * A live stream can leave its slot: export its complete state as a blob, import the blob into any slot of any batch of
 * the same plan (another batch, another GPU, another process), and the stream continues there bit for bit, with no
 * restart and no new latency ramp.  Grow or compact a batch, rebalance or drain a device, survive a restart, hand a
 * stream to another worker.
 *
 * Blob (little-endian, format version 1, r8bgpu_plan_state_bytes(plan) bytes, a multiple of 8), in 64-bit words:
 *   - magic "R8BS" and the format version; a checksum of every other word; the blob's length;
 *   - the plan's fingerprint: src, dst, MaxInLen, extfft, trans band, atten, fasttiming, the stage count, max_trim, and a
 *     hash of the designed stage data (filters, banks, ratios, timing);
 *   - pass_n (passthrough plans), the trim factor, the dither setting, and the count of dithered outputs m;
 *   - per stage: input and output totals, the order-2 interpolator's timing state (with its dsr), and H_j;
 *   - the 16-slot dither error history;
 *   - for every stage input j, the window [n_in_j - H_j, n_in_j) of that stream as fp64 (negative indices stored as 0).
 *     H_j depends on the plan only (r8bgpu_plan_state_windows): the longest reach any batch of the plan may re-read,
 *     src_history plus what refilling a link that lock-step calls keep in shared memory needs, capped by the ring a batch
 *     keeps.  A few tens of KB per channel for MaxInLen 65536.
 * Semantics:
 *   - Export changes no output.  A lock-step batch whose link rings are stale first runs the refill a ragged call would
 *     run (allocating the link rings once), so the blob does not depend on the exporter's fusion.
 *   - Import acts like r8bgpu_batch_clear_channels on the slot followed by installing the exported state: its schedule
 *     joins an equal group or gets its own, and the slot carries the exported trim factor and dither setting.  A target
 *     whose links are stale refills its own channels first; the imported windows are the exporter's bits, never
 *     recomputed.  Other channels are untouched; a batch whose channels all end in one state runs lock-step again.
 *   - Refused, changing nothing, each with its own message: a format or fingerprint mismatch, a bad checksum or a
 *     truncated blob (stride_bytes below the plan's blob size), a channel out of range or named twice, an R8B_FASTTIMING
 *     plan (it runs lock-step only), and on a mixed batch a channel whose plan differs from the blob's.
 *   - Routing: R8BGPU_DEVICE_ALL batches send channel ranges to their shards (host forms only), mixed batches send each
 *     channel to its part and keep the dither state themselves.
 * r8bgpu_batch_export / _import: blob i for channels[i] at buf + i * stride_bytes in host memory (stride_bytes at least
 * the largest blob of the named channels' plans).  r8bgpu_batch_export_device / _import_device: the same bytes in device
 * memory on the batch's GPU, 8-byte aligned, for moves on one GPU without crossing PCIe.  All four finish before they
 * return, like r8bgpu_batch_clear_channels. */
R8BGPU_API size_t r8bgpu_plan_state_bytes(const r8bgpu_plan* plan);
/* H_j of every stage input j into windows[0 .. cap); returns the stage count. */
R8BGPU_API int r8bgpu_plan_state_windows(const r8bgpu_plan* plan, long long* windows, int cap);
/* The plan's fingerprint as a blob stores it (min(cap, 64) bytes into out); returns its length, 64. */
R8BGPU_API int r8bgpu_plan_state_fingerprint(const r8bgpu_plan* plan, void* out, int cap);
R8BGPU_API int r8bgpu_batch_export(r8bgpu_batch* batch, const int* channels, int n, void* buf, size_t stride_bytes);
R8BGPU_API int r8bgpu_batch_import(r8bgpu_batch* batch, const int* channels, int n, const void* buf, size_t stride_bytes);
R8BGPU_API int r8bgpu_batch_export_device(r8bgpu_batch* batch, const int* channels, int n, void* buf, size_t stride_bytes);
R8BGPU_API int r8bgpu_batch_import_device(r8bgpu_batch* batch, const int* channels, int n, const void* buf,
                                          size_t stride_bytes);

/* ---- long clips --------------------------------------------------------------------------
 * CDSPResampler::oneshot() (CDSPResampler.h:592-651) of whole clips on the whole GPU: a batch of n_ch channels is used as
 * n_ch lanes, and one call resamples n_clips clips, each cut into time segments that run side by side.  Clip r's output
 * is exactly, bit for bit in fp64 and byte for byte in typed outputs, what a one-channel batch of the same plan returns
 * when the clip goes in as blocks of B samples from sample 0 (B = MaxInLen, rounded down to a multiple of 8 for DSD input)
 * followed by a flush to oplens[r]: the "twin" run.
 *   - Segments start at multiples P_k of B.  The lane of a segment starts W samples earlier (at S_k = max(0, P_k - W)) in
 *     the twin's schedule state after S_k / B blocks (every stage's totals and the order-2 interpolator's timing state),
 *     with zeroed rings, and is fed the twin's own blocks from S_k on.  It keeps the absolute outputs [E(P_k), E(P_k+1)),
 *     E(P) = the twin's output total after P inputs; a clip's last segment ends with a flush to oplens[r].  Nothing at or
 *     past oplens[r] is kept, and segments that keep nothing do not run.
 *   - W (r8bgpu_plan_oneshot_warmup) is long enough that at P_k every ring window a later call can read holds the twin's
 *     bits: the zeros before S_k taint one overlap-save tile plus the filter's reach per stage (DESIGN.md section 10).
 *   - Scheduling: the call runs in rounds of ragged calls; in each, every lane of the round advances by one block (or
 *     idles), then the round's last segments flush.  Layout policy (r8bgpu_plan_simulate_oneshot): with m clips that keep
 *     output, R = ceil(m / n_lanes) rounds at least; the segment length is the fewest blocks that fits every clip's
 *     segments into R * n_lanes lanes; segments are sorted by length (longest first) and dealt out n_lanes per round.
 * Arguments:
 *   - Clip r is row r of a planar buffer (data + r * stride, stride at least its length in elements) or column r of an
 *     interleaved one (stride at least n_clips).  Inputs: every format of the typed ragged calls (DSD lengths multiples of
 *     8); outputs: every non-DSD format.
 *   - lens / oplens: 64-bit sample counts; oplens NULL: each clip's ceil(lens[r] * dst / src).
 *   - dither: NULL (the plain cast) or one setting per clip, kind OFF or TPDF with n_taps == 0.  Integer output n of clip
 *     r takes steps 1-5 of the dither contract (r8bgpu_batch_set_dither) with that index.  Noise shaping is refused: its
 *     error feedback runs through the whole clip.
 * Both forms clear every lane first, leave the batch cleared and finish before they return; the lanes' own dither and
 * trim settings are neither used nor changed.  The host form holds no device memory proportional to a clip: each call's
 * lane blocks cross PCIe through the batch's staging blocks.  Passthrough plans return the converted copy, zero-padded
 * to oplens.  Refused, changing nothing, each with its own message: mixed and R8BGPU_DEVICE_ALL batches, trim / asrc
 * plans, R8B_FASTTIMING plans, a batch with DSD output on, shaped dither, negative lengths, buffers too short for their
 * lengths, DSD lengths that are not multiples of 8.  The dry run refuses the same plans. */
typedef struct r8bgpu_oneshot_seg {
    int clip;
    int lane, round;
    int pad_;
    long long start;          /* S_k: the lane's first input sample */
    long long p0, p1;         /* P_k, P_k+1: the input samples whose outputs it keeps */
    long long e0, e1;         /* the kept absolute outputs [e0, e1) */
} r8bgpu_oneshot_seg;
/* W of the plan: input samples each segment re-reads before its first kept output (a multiple of MaxInLen). */
R8BGPU_API long long r8bgpu_plan_oneshot_warmup(const r8bgpu_plan* plan);
/* Dry run (no GPU): the segment layout a batch of n_lanes lanes would use, with B = MaxInLen: the layout of every input
 * format when MaxInLen is a multiple of 8 (DSD input otherwise runs in blocks of MaxInLen rounded down to one).  Returns the number of segments
 * that run; *n_calls = ragged calls, one per round's flush included; seg (may be NULL) receives the first cap of them, by
 * round and lane. */
R8BGPU_API int r8bgpu_plan_simulate_oneshot(const r8bgpu_plan* plan, int n_lanes, int n_clips, const long long* lens,
                                            const long long* oplens, int* n_calls, r8bgpu_oneshot_seg* seg, int cap);
R8BGPU_API int r8bgpu_batch_oneshot(r8bgpu_batch* batch, const r8bgpu_buffer* d_in, int n_clips, const long long* lens,
                                    const r8bgpu_buffer* d_out, const long long* oplens, const r8bgpu_dither* dither);
R8BGPU_API int r8bgpu_batch_oneshot_host(r8bgpu_batch* batch, const r8bgpu_buffer* h_in, int n_clips,
                                         const long long* lens, const r8bgpu_buffer* h_out, const long long* oplens,
                                         const r8bgpu_dither* dither);

/* ---- gradients through long clips ----------------------------------------------------------
 * For a plan, a clip of len samples and oplen outputs, let A be the oplen x len matrix of the twin run above in exact
 * arithmetic: the clip in blocks of MaxInLen from sample 0, then the flush to oplen, with the twin's own order-2 read
 * positions and fractions (per-call re-bases and flush sub-steps included).  The zeros the flush feeds are constants.
 * r8bgpu_batch_oneshot_adjoint returns x = A^T g for every clip in one call: g is row r of d_gout (oplens[r] samples),
 * x is row r of d_gin (lens[r] samples; nothing past lens[r] is written).  A passthrough plan returns g cut or
 * zero-padded to lens[r].  oplens NULL: the default targets of r8bgpu_batch_oneshot.
 *   - The transposed chain runs stage by stage in reverse over whole streams: each stage's transpose is a gather, one
 *     thread per gradient sample summing its terms in a fixed order, so the bytes do not depend on the batch's lane
 *     count, the clip's index or neighbours, the layout, the stride or repetition.  No atomics.
 *   - Buffers are R8BGPU_F64 or R8BGPU_F32 with scale 1, planar or interleaved, as for r8bgpu_batch_oneshot.
 *   - The batch gives the device and stream only; its lanes, dither and trim settings are not touched.  The call's
 *     scratch (r8bgpu_plan_oneshot_adjoint_bytes) is allocated on the batch stream and freed before it returns, and the
 *     call finishes before it returns.
 *   - Refused, changing nothing, each with its own message: everything r8bgpu_batch_oneshot refuses, buffers of any other
 *     format or scale, negative lengths, buffers too short for their lengths, and scratch that cannot be allocated. */
R8BGPU_API int r8bgpu_batch_oneshot_adjoint(r8bgpu_batch* batch, const r8bgpu_buffer* d_gout, int n_clips, const long long* lens,
                                            const long long* oplens, const r8bgpu_buffer* d_gin);
/* R_j for each stage j (no GPU): one past the largest index of stage j's input stream that an output in [0, oplen) reads
 * through the chain.  Writes the first cap of them; returns the stage count, < 0 on error. */
R8BGPU_API long long r8bgpu_plan_oneshot_adjoint_extents(const r8bgpu_plan* plan, long long len, long long oplen, long long* ext,
                                                         int cap);
/* Bytes of device scratch r8bgpu_batch_oneshot_adjoint allocates for these clips (its stage tables aside); < 0 on error. */
R8BGPU_API long long r8bgpu_plan_oneshot_adjoint_bytes(const r8bgpu_plan* plan, int n_clips, const long long* lens,
                                                       const long long* oplens);

/* ---- long clips at mixed rates -------------------------------------------------------------
 * Long clips and their gradients on a mixed batch (r8bgpu_batch_create_mixed): clip r runs plans[plan_of_clip[r]], the
 * plan index r8bgpu_batch_part takes.  On an ordinary batch every index must be 0, and the calls are exactly
 * r8bgpu_batch_oneshot / _oneshot_host / _oneshot_adjoint.
 *   - Clip r behaves exactly as on an ordinary batch of its plan: its forward output is that plan's twin run, bit for bit
 *     in fp64 and byte for byte in typed outputs (flat TPDF included), and its gradient is that plan's A^T g, bit for bit.
 *     oplens NULL: ceil(lens[r] * dst / src) of the clip's own plan.
 *   - Clip indices stay the caller's: row or column r of every buffer, dither[r], and the messages that name a clip.
 *     Formats, layouts, strides and scales are those of r8bgpu_batch_oneshot, DSD input and passthrough parts included
 *     (DSD64 and DSD128 clips to 88200 in one call; 16 kHz clips on a 16 kHz part return the converted copy).
 *   - Lanes: the clips of plan p run on part p's channels only, laid out by the long-clip policy with that part's lane
 *     count, so r8bgpu_plan_simulate_oneshot(plans[p], lanes of p, the clips of p in the caller's order) is the dry run
 *     of part p.  A part that no clip names runs nothing.
 *   - Streams: an event recorded on the batch stream makes every part's stream wait for the work queued there (the
 *     input is often produced on it), each part runs on its own stream, and the batch stream waits for every part.  The
 *     forward issues the parts' ragged calls round-robin, one call per part at a time, so a part waiting for its upload
 *     (host form) does not hold back the others' issue.  The adjoint runs each plan's transposed chain on its part's
 *     stream, with that group's scratch allocated and freed there.  Every form finishes before it returns.
 *   - The whole mixed batch is cleared before and after the forward, as by r8bgpu_batch_clear (its dither streams
 *     included); the lanes' trim and dither settings are neither used nor changed.
 *   - Refused, changing nothing (every check runs before any part runs), each with its own message: what
 *     r8bgpu_batch_oneshot / _oneshot_adjoint refuse, judged per named plan (trim / asrc parts and R8B_FASTTIMING plans;
 *     a trim part that no clip names is fine), DSD output on, shaped dither, negative lengths, short strides, a plan
 *     index out of range, a null plan_of_clip with n_clips > 0, and R8BGPU_DEVICE_ALL batches. */
R8BGPU_API int r8bgpu_batch_oneshot_mixed(r8bgpu_batch* batch, const r8bgpu_buffer* d_in, int n_clips, const int* plan_of_clip,
                                          const long long* lens, const r8bgpu_buffer* d_out, const long long* oplens,
                                          const r8bgpu_dither* dither);
R8BGPU_API int r8bgpu_batch_oneshot_mixed_host(r8bgpu_batch* batch, const r8bgpu_buffer* h_in, int n_clips,
                                               const int* plan_of_clip, const long long* lens, const r8bgpu_buffer* h_out,
                                               const long long* oplens, const r8bgpu_dither* dither);
R8BGPU_API int r8bgpu_batch_oneshot_adjoint_mixed(r8bgpu_batch* batch, const r8bgpu_buffer* d_gout, int n_clips,
                                                  const int* plan_of_clip, const long long* lens, const long long* oplens,
                                                  const r8bgpu_buffer* d_gin);

/* ---- crops of long clips -------------------------------------------------------------------
 * A crop {clip r, o0, o1} asks for the outputs [o0, o1) of clip r's twin run (see "long clips") with target oplens[r],
 * 0 <= o0 <= o1 <= oplens[r] (oplens NULL: ceil(lens[r] * dst / src) of the clip's plan).  Crop k's output is elements
 * [o0, o1) of what r8bgpu_batch_oneshot returns for that clip, bit for bit in fp64 and byte for byte in typed outputs
 * (flat TPDF included: the dither index is the absolute output index), whatever the call's other crops, their order,
 * the lane count, the buffer layout or whether the batch is mixed.  Crops may name the same clip, overlap, be empty and
 * reach into the flush tail.
 *   - Layout: each crop is a span of its clip's twin.  It starts at P_lo, the first multiple of B below lens[r] (or 0)
 *     whose E is the largest E(P) <= o0 (so a crop from output 0 starts at 0, laid out as the whole clip), and ends at the first multiple of B (or lens[r]) with E >= o1; only when o1 > E(lens[r]) does
 *     it end in the twin's flush, and that flush runs to oplens[r], not to o1 (a flush's outputs depend on its
 *     sub-steps, so only the twin's own target gives the twin's bits).  Segments are cut from P_lo by the long-clip
 *     policy, each starting W earlier in the twin's state, and keep only [o0, o1).  All crops of a clip share the walks
 *     of its twin on the host.  r8bgpu_plan_simulate_oneshot_crops is the dry run; its segments carry the CROP index in
 *     `clip`.
 *   - plan_of_clip: NULL on an ordinary batch (or every index 0); on a mixed batch one plan index per clip, and each
 *     crop runs on the part of its clip's plan, as in r8bgpu_batch_oneshot_mixed.
 *   - Forward output: crop k is row k of d_out (planar: stride at least max(o1 - o0)) or column k (interleaved: stride
 *     at least n_crops); element i is output o0 + i, and nothing past o1 - o0 is written.  Input buffers, formats,
 *     scales, DSD input and dither (dither[clip]) are those of r8bgpu_batch_oneshot.
 *   - Adjoint: for each crop k, x_k = A[o0:o1, :]^T g_k with A the clip's twin map (see "gradients through long clips")
 *     and g_k row or column k of d_gout.  Every clip that a crop names gets, in its row or column of d_gin, the sum of
 *     its crops' x_k in ascending crop index over the hull [min lo_0, max hi_0) of their input windows, clipped to
 *     [0, lens[clip]); hull samples that no crop reaches are set to 0.  Nothing else of d_gin is written: zero it first.
 *     Each crop's transposed chain runs over its windows only (scratch rows as wide as the widest window), so the work
 *     follows the crops' lengths, not the clips'.  Buffers are F64 or F32 with scale 1.
 *   - r8bgpu_plan_oneshot_crop_extents (no GPU): for each stage input j, the window [lo_j, hi_j) of samples that any
 *     output in [o0, o1) of a clip of len samples and target oplen reads through the chain.  hi_j is
 *     r8bgpu_plan_oneshot_adjoint_extents' R_j with oplen = o1; on a block-exact stage lo_j is the window start of the
 *     first block holding a needed output; a half-band decimator's lo_j is even.  An empty crop has empty windows
 *     [0, 0).  Writes the first cap of each; returns the stage count, < 0 on error.
 *   - Refused, changing nothing, with the long-clip calls' messages: trim / asrc plans, R8B_FASTTIMING plans, DSD
 *     output on, shaped dither, R8BGPU_DEVICE_ALL batches, negative lengths, short input strides.  In addition, each
 *     with its own message: a crop whose clip is out of range, o0 < 0, o1 < o0, o1 > oplens[clip], null crops with
 *     n_crops > 0, and output strides shorter than the longest crop (or, interleaved, than n_crops). */
typedef struct r8bgpu_crop {
    int clip;            /* row / column of the input buffer; index into lens, oplens, plan_of_clip, dither */
    int pad_;
    long long o0, o1;    /* outputs [o0, o1) of the clip's twin run */
} r8bgpu_crop;
R8BGPU_API int r8bgpu_batch_oneshot_crops(r8bgpu_batch* batch, const r8bgpu_buffer* d_in, int n_clips, const int* plan_of_clip,
                                          const long long* lens, const long long* oplens, int n_crops,
                                          const r8bgpu_crop* crops, const r8bgpu_buffer* d_out, const r8bgpu_dither* dither);
R8BGPU_API int r8bgpu_batch_oneshot_crops_host(r8bgpu_batch* batch, const r8bgpu_buffer* h_in, int n_clips,
                                               const int* plan_of_clip, const long long* lens, const long long* oplens,
                                               int n_crops, const r8bgpu_crop* crops, const r8bgpu_buffer* h_out,
                                               const r8bgpu_dither* dither);
R8BGPU_API int r8bgpu_batch_oneshot_crops_adjoint(r8bgpu_batch* batch, const r8bgpu_buffer* d_gout, int n_clips,
                                                  const int* plan_of_clip, const long long* lens, const long long* oplens,
                                                  int n_crops, const r8bgpu_crop* crops, const r8bgpu_buffer* d_gin);
R8BGPU_API int r8bgpu_plan_simulate_oneshot_crops(const r8bgpu_plan* plan, int n_lanes, int n_clips, const long long* lens,
                                                  const long long* oplens, int n_crops, const r8bgpu_crop* crops,
                                                  int* n_calls, r8bgpu_oneshot_seg* seg, int cap);
R8BGPU_API long long r8bgpu_plan_oneshot_crop_extents(const r8bgpu_plan* plan, long long len, long long oplen, long long o0,
                                                      long long o1, long long* lo, long long* hi, int cap);

/* Number of kernels this batch has launched since creation. */
R8BGPU_API unsigned long long r8bgpu_batch_kernel_launches(const r8bgpu_batch* batch);
/* Per-stage device timing for profiling/bench: when enabled every stage launch is bracketed
 * by CUDA events on the batch's stream.  r8bgpu_batch_stage_time_ms() synchronises and returns the
 * accumulated milliseconds (and launch count) of one stage since timing was (re-)enabled.  Stage index
 * r8bgpu_plan_stage_count(plan) is the DSD output modulator (r8bgpu_batch_set_dsd_out). */
R8BGPU_API int r8bgpu_batch_set_timing(r8bgpu_batch* batch, int enable);
R8BGPU_API double r8bgpu_batch_stage_time_ms(r8bgpu_batch* batch, int stage, unsigned long long* launches);
/* Name of the kernel that executes plan stage `stage`; returns the number of consecutive plan stages
 * that kernel covers (0: the stage is folded into an earlier stage's kernel), < 0 on error. */
R8BGPU_API int r8bgpu_batch_stage_kernel(const r8bgpu_batch* batch, int stage, char* name, int cap);
/* The instantiation of the fused kernel the last lock-step call launched for plan stage `stage` (the BlockConvolver
 * of a fused pair, or a 2x BlockConvolver on k_up2_frac2), with its template arguments in declaration order:
 * "k_up2_frac2<IR,PAD,GLOG,TC,UP,COPY,POLY,CS,LIN> mbu=N" or "k_up2_frac<MODE,IR,PAD,BANK>", e.g.
 * "k_up2_frac2<8,false,0,true,2,false,false,true,true> mbu=6".  On the first stage of a half-band cascade, the cascade
 * kernel and its tile plan (r8bgpu_plan_cascade_info): "k_hbup_cascade stages=5 taps=11/6/5/4/3 last2=1 w=160" or
 * "k_hbdown_cascade stages=6 taps=2/3/4/5/6/11 w=16" ("k_hbdown_cascade<DSD> ..." where the call read DSD bytes).
 * On an unfused BlockConvolver or interpolator, its kernel with the call's fields (r8bgpu_plan_blockconv_info,
 * r8bgpu_plan_frac_info): "k_blockconv M=2048 up=2 src_up=1 down=3 trunc=0 tiles=6", "k_bcl M=65536 R0=16 src_up=1
 * down=1 trunc=0 tiles=2 groups=2" (tiles of the largest channel group's call, launch groups of channels) or
 * "k_frac poly=1 tile=256 flen=24".  Empty when no such call has launched one since the batch was created.  Returns the length of the text (written up
 * to cap - 1 bytes), < 0 on error. */
R8BGPU_API int r8bgpu_batch_last_variant(const r8bgpu_batch* batch, int stage, char* name, int cap);
/* Bytes of device memory held by the batch (state rings + tables + staging). */
R8BGPU_API unsigned long long r8bgpu_batch_device_bytes(const r8bgpu_batch* batch);

/* Calibration for the bench's secondary (fp64) roofline: measured DFMA throughput of `device` (< 0: current) in
 * TFLOP/s, register-resident, ~10 ms; < 0 on error.  Replaces nothing in the reference. */
R8BGPU_API double r8bgpu_measure_fp64_tflops(int device);

/* Page-locked host memory for the *_host entry points (optional but faster). */
R8BGPU_API void* r8bgpu_host_alloc(size_t bytes);
R8BGPU_API void r8bgpu_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif /* R8BGPU_H_INCLUDED */

// r8b_capi.cu -- the engine behind include/r8bgpu.h: device-resident per-channel state, the
// per-call launch sequence, and the extern "C" boundary.
//
// Per-channel state in HBM (SURVEY.md appendix C), all planar [channel][...]:
//   * input history ring      : the most recent source samples the first stage may re-read
//   * one ring per stage link : the stream between stage i and i+1, absolute-indexed,
//                               capacity = pow2 >= (max samples per call + look-back of stage i+1)
// Shared read-only per plan: filter spectrum (slot order, pre-scaled), FFT twiddles, fractional
// delay bank.  All integer scheduling state lives on the host (Schedule): once per batch, or once per group of
// channels in the same state after ragged calls / per-channel clears (RaggedSchedule).
#include "../../include/r8bgpu.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <string>
#include <utility>
#include <vector>

#include "r8b_bclarge.cuh"
#include "r8b_codec.cuh"
#include "r8b_dither.cuh"
#include "r8b_dsd.cuh"
#include "r8b_dsdmod.cuh"
#include "r8b_fft.cuh"
#include "r8b_hosttab.h"
#include "r8b_kernels.h"
#include "r8b_multi.h"
#include "r8b_plan.h"

using namespace r8bgpu;

namespace {

thread_local std::string g_err;

void set_err(const std::string& s) { g_err = s; }

bool cuda_ok(cudaError_t e, const char* what)
{
    if (e == cudaSuccess) return true;
    g_err = std::string(what) + ": " + cudaGetErrorString(e);
    return false;
}

long long next_pow2(long long v)
{
    long long p = 1;
    while (p < v) p <<= 1;
    return p;
}

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev)
    {
        if (cudaGetDevice(&prev) != cudaSuccess) {
            ok = false;
            return;
        }
        if (prev != dev) ok = (cudaSetDevice(dev) == cudaSuccess);
    }
    ~DeviceGuard()
    {
        int cur = -1;
        if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
    }
};

// One device block (or, Pinned, one page-locked host block) of n T's, freed by reset() and by its destructor.  A device
// block is charged to a byte counter -- its batch's dev_bytes -- for as long as it is held; nothing else writes that
// counter, so it always equals the device memory the batch holds.
template <class T, bool Pinned = false>
class Buf {
  public:
    Buf() = default;
    Buf(Buf&& o) noexcept { *this = std::move(o); }
    Buf& operator=(Buf&& o) noexcept
    {
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
        std::swap(charge_, o.charge_);
        return *this;
    }
    ~Buf() { reset(); }
    operator T*() const { return p_; }
    size_t size() const { return n_; }
    void reset()
    {
        if (p_ == nullptr) return;
        if (Pinned) cudaFreeHost(p_);
        else cudaFree(p_);
        if (charge_ != nullptr) *charge_ -= n_ * sizeof(T);
        p_ = nullptr;
        n_ = 0;
    }
    // device blocks: a new block of n
    bool alloc(unsigned long long& charge, size_t n, const char* what) { return take(n, what, &charge); }
    // ... at least n, the block held if it is large enough
    bool grow(unsigned long long& charge, size_t n, const char* what) { return n <= n_ || take(n, what, &charge); }
    // ... a new block holding v
    bool upload(unsigned long long& charge, const std::vector<T>& v, const char* what, const char* copy_what)
    {
        return take(v.size(), what, &charge) &&
               cuda_ok(cudaMemcpy(p_, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice), copy_what);
    }
    // pinned host blocks (not charged)
    bool alloc(size_t n, const char* what) { return take(n, what, nullptr); }
    bool grow(size_t n, const char* what) { return n <= n_ || take(n, what, nullptr); }

  private:
    bool take(size_t n, const char* what, unsigned long long* charge)
    {
        reset();
        void* p = nullptr;
        if (!cuda_ok(Pinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T)), what)) return false;
        p_ = static_cast<T*>(p);
        n_ = n;
        charge_ = charge;
        if (charge_ != nullptr) *charge_ += n * sizeof(T);
        return true;
    }
    T* p_ = nullptr;
    size_t n_ = 0;
    unsigned long long* charge_ = nullptr;
};
template <class T>
using DevBuf = Buf<T>;
template <class T>
using PinBuf = Buf<T, true>;

// An owned CUDA event or stream, destroyed with its owner.
template <class H, cudaError_t (*Destroy)(H)>
class Handle {
  public:
    Handle() = default;
    Handle(Handle&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    Handle& operator=(Handle&& o) noexcept
    {
        std::swap(h_, o.h_);
        return *this;
    }
    ~Handle() { reset(); }
    operator H() const { return h_; }
    void reset()
    {
        if (h_ != nullptr) Destroy(h_);
        h_ = nullptr;
    }
    // for the call that creates the handle: the one held is released first
    H* put()
    {
        reset();
        return &h_;
    }

  private:
    H h_ = nullptr;
};
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;

// Per-call records that go up to one device array from two pinned host arrays in turn, so that the host fills one while
// the other's copy may still be queued.  next() hands out the other host array once its last upload has finished;
// upload() copies part of the current one up in stream order (a call may upload several parts).
template <class T>
struct RecRing {
    DevBuf<T> d;
    PinBuf<T> h[2];
    Event ev[2];
    int cur = 0;

    bool create(unsigned long long& charge, size_t n, const char* dev_what, const char* host_what, const char* ev_what)
    {
        if (!d.alloc(charge, n, dev_what)) return false;
        for (int k = 0; k < 2; k++)
            if (!h[k].alloc(n, host_what) || !cuda_ok(cudaEventCreateWithFlags(ev[k].put(), cudaEventDisableTiming), ev_what))
                return false;
        return true;
    }
    T* next(const char* what)
    {
        cur ^= 1;
        return cuda_ok(cudaEventSynchronize(ev[cur]), what) ? (T*) h[cur] : nullptr;
    }
    T* host() const { return h[cur]; } // the array next() handed out last
    bool upload(size_t first, size_t n, cudaStream_t st, const char* what)
    {
        return cuda_ok(cudaMemcpyAsync(d + first, h[cur] + first, n * sizeof(T), cudaMemcpyHostToDevice, st), what) &&
               cuda_ok(cudaEventRecord(ev[cur], st), what);
    }
};

struct StageDev {
    // BLOCKCONV
    int fft_log2 = 0, lg = 0, virt_up = 1;
    double nyq_gain = 0.0;
    DevBuf<double2> spec;
    DevBuf<double2> tw;
    // large-tile path (r8b_bclarge.cuh): W_M table and the scratch buffer, which holds scratch_pairs tile pairs of M points
    bool large = false;
    DevBuf<double2> tw_m;
    DevBuf<double2> scratch;
    long long scratch_pairs = 0;
    // FRAC
    DevBuf<double> bank;
    int frac_tile_fixed = 0;  // k_frac outputs per CTA of every call; 0: sized per call from its ratio (trim plans)
    int frac_tile_ragged = 0; // ... of ragged calls
    std::string unfused_variant; // k_blockconv, the large-tile trio or k_frac as the last lock-step call launched it
    // source ring of this stage (for stage 0: the input history ring)
    DevBuf<double> ring;
    long long ring_cap = 0;
    // fusion: a 2x BLOCKCONV immediately followed by a FRAC stage runs as ONE kernel
    bool fused_with_next = false; // on the BLOCKCONV stage
    bool fused_into_prev = false; // on the FRAC stage (its source ring is never materialised)
    DevBuf<int> phase_off;
    DevBuf<int> phase_row;
    DevBuf<double> gbank; // whole stepping: grouped, pre-shifted, zero-padded bank (see FusedParams)
    DevBuf<int> goff;
    int gbank_len = 0, gbank_smem_len = 0, smaxp = 0, ir = 8;
    int yl = 0, yr = 0, ysh = 31, span_max = 0, bank_in_smem = 0;
    // R8B_FASTTIMING position tables (FRAC_POLY stages of fast-timing plans)
    RecRing<int> ft_dp;
    RecRing<double> ft_fpos;
    int casc_len = 0; // >= 2 on the first stage of a run of HBUP stages executed by k_hbup_cascade
    HbCascadeParams up_casc; // its tile plan (taps, halos, shared-memory layout)
    int up_casc_smem = 0;
    int down_casc_len = 0; // >= 2 on the first stage of a run of HBDOWN stages executed by k_hbdown_cascade
    HbDownCascParams down_casc; // its tile plan
    int down_casc_smem = 0;
    int casc_variant = 0; // the cascade kernel the last lock-step call launched: 1, or 2 for k_hbdown_cascade<DSD>
    // v2 fused kernel (r8b_fused2.cu): [q][r] twiddle tables for the bulk copy; on the BLOCKCONV stage
    DevBuf<double2> tw_tab;
    DevBuf<double2> c_tab;    // v2 fused kernel: phase C operands in thread order
    DevBuf<double2> cd_tab;   // v2 fused kernel, up 2: operands of phase C fused into the first inverse pass
    DevBuf<double2> cs_tab;   // the same spectrum in its symmetric half-size form, when the plan has room for it in shared memory
    DevBuf<double2> c_tab_v1; // round-1 fused kernel: its two spectrum values per frequency pair in thread order
    bool bank_frag_order = false; // grouped bank stored in mma fragment order (only the tensor-path interpolation reads it)
    bool f2_ok = false;
    bool f2_poly = false; // order-2 interpolator on the v2 kernel's tensor path (decided per call: near-integer ratios)
    bool f2_copy = false; // BlockConvolver 2/1 alone on the v2 kernel (phase E copies the 2x stream out)
    FusedGeom fgeom;
    FusedVariant last_variant; // the fused kernel's instantiation the last lock-step call launched (on the BLOCKCONV stage)
};

// The settings r8bgpu_batch_create reads for the fused kernels (R8BGPU_IR is read by choose_group_ir).
struct FusedKnobs {
    int f2_flags = 6;          // R8BGPU_F2_FLAGS (see r8bgpu_batch::f2_flags)
    bool f2_flags_env = false; // ... set: its flags are used as given
    bool v1 = false;           // R8BGPU_FUSED_V1: no pair on the v2 kernel
    bool no_fusion = false;    // R8BGPU_NO_FUSION: every stage on its own kernel
    bool poly_v2 = false;      // R8BGPU_POLY_V2: order-2 pairs may run on the v2 kernel
};

FusedKnobs fused_knobs_env()
{
    FusedKnobs k;
    if (const char* e = getenv("R8BGPU_F2_FLAGS")) {
        k.f2_flags = atoi(e);
        k.f2_flags_env = true;
    }
    k.v1 = getenv("R8BGPU_FUSED_V1") != nullptr;
    k.no_fusion = getenv("R8BGPU_NO_FUSION") != nullptr;
    k.poly_v2 = getenv("R8BGPU_POLY_V2") != nullptr;
    return k;
}

// How a batch runs BlockConvolver stage i of a plan with the interpolator behind it: whether the two fuse, on which
// kernel, with which bank layout, and the geometry of both whole-stepping bank layouts.  r8bgpu_batch_create acts on
// it and r8bgpu_plan_fused_info reports it, so a test can see every decision without a device.
struct FusedPlan {
    FusedGeom geom;              // geom.ok: stage i + 1 runs inside stage i's kernel
    bool copy = false;           // a 2x BlockConvolver alone on k_up2_frac2 (phase E copies the 2x stream out)
    bool poly_v2 = false;        // fused with an order-2 interpolator that may run on k_up2_frac2 (decided per call)
    bool cs = false;             // up 2 on k_up2_frac2: the symmetric spectrum table fits beside the largest bank
    bool whole = false;          // stage i + 1 is a whole-stepping interpolator: tc and fma below are its banks
    GroupBank tc, fma;           // its bank in the tensor-path layout (8 phases, fragment order) and the FMA layout
    bool tc_fits = false, fma_fits = false; // k_up2_frac2 can hold that bank (shared memory, at most 192 groups)
    bool tc_bank = false;        // the fused pair loads the tensor-path bank (else the FMA one)
    bool bank_in_smem = false;   // k_up2_frac: the bank it loads fits its shared memory
    int kernel = R8BGPU_FUSED_NONE;
};

FusedPlan plan_fused_stage(const std::vector<StageDesc>& st, size_t i, const FusedKnobs& k)
{
    FusedPlan fp;
    const StageDesc& s = st[i];
    if (s.kind != ST_BLOCKCONV) return fp;
    fp.whole = i + 1 < st.size() && st[i + 1].kind == ST_FRAC_WHOLE;
    if (fp.whole) {
        const StageDesc& f = st[i + 1];
        auto f2_fits = [](const GroupBank& gb) {
            return fused2_smem_bytes(gb.n_groups * gb.smaxp * gb.ir, false, false) <= kFused2SmemMax && gb.n_groups <= 192;
        };
        fp.tc = build_group_bank(f, 8, true);
        fp.fma = build_group_bank(f, choose_group_ir(f), false);
        fp.tc_fits = f2_fits(fp.tc);
        fp.fma_fits = f2_fits(fp.fma);
    }
    // Fusable pair: [BlockConv 2/1 or 1/1 with a kernel that fits M=4096 tiles] -> [FracInterp].  The 1x pair exists only
    // in the v2 kernel with the tensor-path interpolation: its bank must fit.
    if (i + 1 < st.size() && !k.no_fusion) {
        fp.geom = fused_geometry(s, st[i + 1]);
        if (fp.geom.ok && fp.geom.up == 1 && (k.v1 || !(k.f2_flags & 4) || !fp.tc_fits)) fp.geom = FusedGeom();
    }
    const bool fused = fp.geom.ok;
    // (opt-in: measured slower than the round-1 kernel's staged-row path, see DESIGN.md section 3)
    if (fused && st[i + 1].kind == ST_FRAC_POLY && fp.geom.up == 2 && (k.f2_flags & 4) && !k.v1 && k.poly_v2 &&
        (st[i + 1].bank.filter_len & 1) == 0 && st[i + 1].bank.filter_len <= 32)
        fp.poly_v2 = true;
    // a 2x BlockConvolver that no interpolator follows runs on the v2 fused kernel too (its phase E copies the stream out)
    // when the polyphase branches fit 4096-point tiles
    if (!fused && s.up == 2 && s.down == 1 && !s.block_exact && !k.no_fusion && !k.v1) {
        const BcTile bt = blockconv_tile(s);
        if (!bt.large && 2 * (4096 - 2 * bt.lg) >= 2048) fp.copy = true;
    }
    // phase C from shared memory where the spectrum pairs fit beside the largest bank this plan can load
    if ((fused && fp.geom.up == 2) || fp.copy) fp.cs = fused2_cs_fits(fused ? fused2_bank_doubles_max(st[i + 1]) : 0);
    if (fused && fp.whole) {
        const bool want_f2 = !k.v1;
        fp.tc_bank = want_f2 && (k.f2_flags & 4) && fp.tc_fits; // else the v1 kernel reads the plain layout
        const GroupBank& B = fp.tc_bank ? fp.tc : fp.fma;
        fp.bank_in_smem = fused_smem_bytes(B.n_groups * B.smaxp * B.ir) <= 220 * 1024;
        // the persistent two-pipeline kernel needs the call's whole bank in shared memory
        if (want_f2 && (fp.tc_bank || fp.fma_fits)) fp.kernel = fp.tc_bank ? R8BGPU_FUSED_F2_TC : R8BGPU_FUSED_F2_FMA;
        else fp.kernel = fp.bank_in_smem ? R8BGPU_FUSED_V1_SMEM : R8BGPU_FUSED_V1_GLOBAL;
    } else if (fused) {
        fp.kernel = R8BGPU_FUSED_ORDER2;
    } else if (fp.copy) {
        fp.kernel = R8BGPU_FUSED_F2_COPY;
    }
    return fp;
}

// The settings r8bgpu_batch_create reads for runs of half-band stages.
struct HbKnobs {
    bool no_cascade = false;   // R8BGPU_NO_FUSION or R8BGPU_NO_HB_CASCADE: one k_hbup / k_hbdown per stage
    bool no_last2 = false;     // R8BGPU_HB_NO_LAST2: the up cascade's last two stages run as two passes
    int up_budget = 7000;      // R8BGPU_HB_SMEM_DOUBLES: doubles of shared memory per up-cascade CTA (4 CTAs of 128 threads per SM; measured best)
    int down_budget = 6400;    // R8BGPU_HBD_SMEM_DOUBLES: doubles per CTA (4 CTAs per SM; measured on 2822400->44100: 3200 0.97, 6400 0.46, 12800 0.53, 25000 0.79 ms)
};

HbKnobs hb_knobs_env()
{
    HbKnobs k;
    k.no_cascade = getenv("R8BGPU_NO_FUSION") != nullptr || getenv("R8BGPU_NO_HB_CASCADE") != nullptr;
    k.no_last2 = getenv("R8BGPU_HB_NO_LAST2") != nullptr;
    if (const char* e = getenv("R8BGPU_HB_SMEM_DOUBLES")) k.up_budget = atoi(e);
    if (const char* e = getenv("R8BGPU_HBD_SMEM_DOUBLES")) k.down_budget = atoi(e);
    return k;
}

// How a batch runs the half-band stage i that no earlier kernel covers: alone (n_stages 1), or with the stages of its
// direction behind it (at most 6 in all) in one cascade kernel with this tile plan.  r8bgpu_batch_create acts on it and
// r8bgpu_plan_cascade_info reports it.
struct HbRunPlan {
    int n_stages = 1;
    HbCascadeParams up;        // n_stages >= 2 of ST_HBUP: the call-independent fields
    HbDownCascParams down;     // n_stages >= 2 of ST_HBDOWN
    int smem_bytes = 0;
};

HbRunPlan plan_hb_run(const std::vector<StageDesc>& st, size_t i, const HbKnobs& k)
{
    HbRunPlan r;
    memset(&r.up, 0, sizeof r.up);
    memset(&r.down, 0, sizeof r.down);
    const StageKind kind = st[i].kind;
    if (k.no_cascade) return r;
    size_t c = 1;
    while (i + c < st.size() && st[i + c].kind == kind && c < 6) c++;
    if (c < 2) return r;
    int* ntaps = kind == ST_HBUP ? r.up.ntaps : r.down.ntaps;
    double(*taps)[14] = kind == ST_HBUP ? r.up.taps : r.down.taps;
    for (size_t s = 0; s < c; s++) {
        ntaps[s] = st[i + s].hb_taps;
        for (int j = 0; j < st[i + s].hb_taps; j++) taps[s][j] = st[i + s].hb[(size_t) j];
    }
    if (kind == ST_HBUP) {
        r.up.n_stages = (int) c;
        r.smem_bytes = hbup_cascade_plan(r.up, k.up_budget, !k.no_last2);
    } else {
        r.down.n_stages = (int) c;
        r.smem_bytes = hbdown_cascade_plan(r.down, k.down_budget);
        if (r.smem_bytes <= 0) { // no tile fits the budget: one k_hbdown per stage
            r.smem_bytes = 0;
            return r;
        }
    }
    r.n_stages = (int) c;
    return r;
}

// Bytes of large-tile scratch a batch may hold for one stage: R8BGPU_BCL_SCRATCH_MB, else 256 MB.  Larger batches run the
// three kernels once per group of channels.
long long bcl_scratch_cap_env()
{
    long long cap = 256LL << 20;
    if (const char* e = getenv("R8BGPU_BCL_SCRATCH_MB")) cap = std::max(1LL, atoll(e)) << 20;
    return cap;
}

// How a batch runs BlockConvolver stage i of a plan with n_ch channels, given its fusion plan fp: the kernel, the tile
// and, on the large path, the scratch.  r8bgpu_batch_create acts on it and r8bgpu_plan_blockconv_info reports it.
struct BcPlan {
    std::string err;             // non-empty: no tile runs this stage
    int kernel = R8BGPU_BC_BLOCKCONV;
    BcTile t;                    // t.fft_log2: the tile the kernel runs (12 on the fused and copy kernels)
    int trunc = 0, adv = 0, smem_bytes = 0;
    int scratch_tiles = 0, group_ch = 0;
    long long scratch_per_ch = 0;
};

BcPlan plan_blockconv_stage(const StageDesc& s, const FusedPlan& fp, int n_ch, long long scratch_cap)
{
    BcPlan bp;
    bp.t = blockconv_tile(s);
    BcTile& t = bp.t;
    if (s.block_exact && t.fft_log2 < 0) {
        // the tile IS the reference's block (2 << BlockLenBits): 64 .. 65536 points for 1x stages (short kernels run on
        // plain radix-2 transforms, blocks above 8192 points on the large-tile path); 2x stages have 1024 .. 4096
        const int lo = t.up == 1 ? 6 : 10, hi = t.up == 1 ? 16 : 12;
        char msg[200];
        snprintf(msg, sizeof msg, "reference-exact decimation needs a %d-point block transform; this build has %d..%d "
                 "points for such stages", 1 << (s.lp.block_len_bits + 1), 1 << lo, 1 << hi);
        bp.err = msg;
        return bp;
    }
    if (fp.copy || fp.geom.ok) {
        bp.kernel = fp.copy ? R8BGPU_BC_F2_COPY : R8BGPU_BC_FUSED;
        t.fft_log2 = 12; // the fused kernels are built for M = 4096
    } else if (t.large) {
        bp.kernel = R8BGPU_BC_LARGE;
    }
    if (t.fft_log2 < 0) {
        bp.err = "low-pass kernel too long for the in-shared-memory FFT tiles";
        return bp;
    }
    const int M = 1 << t.fft_log2;
    bp.trunc = s.block_exact ? s.down : 0;
    bp.adv = s.block_exact ? s.ref_input_len : M - 2 * t.lg;
    if (!t.large) {
        bp.smem_bytes = blockconv_smem_bytes(t.fft_log2, t.up);
        return bp;
    }
    bp.smem_bytes = fft_padded_len(4096) * (int) sizeof(double2);
    // scratch: M complex values per tile pair.  The largest call's input-rate positions [m0, m1) span at most
    // (max_out_len + 2) * D + 2 (for 3x and the zero-stuffed 2x stages: positions of the zero-stuffed stream).
    const long long span = ((long long) s.max_out_len + 2) * s.down + 2;
    long long nt = s.block_exact ? span / s.ref_input_len + 2 : (span + (M - 2LL * t.lg) - 1) / (M - 2LL * t.lg);
    nt += nt & 1;
    bp.scratch_tiles = (int) nt;
    bp.scratch_per_ch = (nt / 2) * M * (long long) sizeof(double2);
    bp.group_ch = (int) std::max(1LL, std::min((long long) n_ch, scratch_cap / bp.scratch_per_ch));
    return bp;
}

// How a batch runs interpolator stage i: on k_frac, the tile of its lock-step calls (whose order-2 ratio a trim plan
// moves per call: tile_fixed is 0 then, unless R8BGPU_FRAC_TILE fixes it) and of its ragged calls.
struct FracPlan {
    std::string err;             // non-empty: R8BGPU_FRAC_TILE is refused
    double in_per_out = 0.0;     // lock-step ratio (a trim plan's at factor 1)
    double in_per_out_ragged = 0.0;
    int tile = 0, tile_ragged = 0;
    int tile_fixed = 0;          // > 0: every call of the batch runs this tile
};

FracPlan plan_frac_stage(const Plan& P, size_t i)
{
    FracPlan f;
    const StageDesc& s = P.stages[i];
    const int flen = s.bank.filter_len;
    const bool trim = (int) i == P.trim_stage;
    f.in_per_out = s.kind == ST_FRAC_WHOLE ? (double) s.in_step / (double) s.out_step : s.src_rate / s.dst_rate;
    f.in_per_out_ragged = s.kind == ST_FRAC_WHOLE ? f.in_per_out : s.src_rate / (trim ? P.trim_dsr(1.0 - P.max_trim) : s.dst_rate);
    f.tile = frac_tile(f.in_per_out, flen);
    f.tile_ragged = frac_tile(f.in_per_out_ragged, flen);
    if (!trim) f.tile_fixed = f.tile;
    if (const char* e = getenv("R8BGPU_FRAC_TILE")) {
        const int v = atoi(e);
        char msg[240];
        if (v < 1 || v > 1024 || (v & (v - 1))) {
            snprintf(msg, sizeof msg, "R8BGPU_FRAC_TILE=%s: need a power of two from 1 to 1024", e);
            f.err = msg;
        } else if (frac_window(v, f.in_per_out_ragged, flen) > FRAC_CAP) {
            snprintf(msg, sizeof msg, "R8BGPU_FRAC_TILE=%d: stage %d (%.17g input samples per output, filter length %d) "
                     "would stage up to %d samples, more than the %d its kernel holds", v, (int) i, f.in_per_out_ragged,
                     flen, frac_window(v, f.in_per_out_ragged, flen), FRAC_CAP);
            f.err = msg;
        }
        f.tile = f.tile_ragged = f.tile_fixed = v;
    }
    return f;
}

} // namespace

struct r8bgpu_plan {
    Plan p;
};

// A multi-device batch (r8bgpu_batch_create(plan, n, -1) on a box with several GPUs) is a FRONT: it owns no device
// state, only one ordinary single-device batch per shard (contiguous channel ranges) and the worker threads that
// drive them side by side (r8b_multi.h).
struct ShardFront {
    std::vector<std::unique_ptr<r8bgpu_batch>> shards;
    std::vector<int> ch0, device, numa;
    std::unique_ptr<ShardPool> pool;
};

// A mixed batch (r8bgpu_batch_create_mixed): channel c is an independent stream of plan plan_of[c].  It owns one ordinary
// single-plan batch per plan (a part, holding that plan's channels in ascending order) and runs each part's ragged chain
// on the part's own fp64 staging rows and stream.  The caller's buffers meet those rows in two mapped conversions
// (r8b_format.cu, MAP) on the batch stream, one in front of the parts and one behind them.
struct MixedFront {
    std::vector<std::unique_ptr<r8bgpu_batch>> parts;
    std::vector<int> part_of, row_of;    // per channel: its part and its row there
    std::vector<std::vector<int>> chans; // per part: its channels, ascending
    int max_out = 0, flush_max_out = 0;  // the largest max_out_len / flush_max_out_len of the plans
    std::vector<Stream> streams;         // per part (the part borrows it as its stream)
    std::vector<Event> done;             // per part: its work of the current call is queued before this
    Event fork;
    RecRing<MapRec> map; // per-call records [2][channel] (in, out), uploaded in one copy
    // host forms: the caller's samples as they cross PCIe
    DevBuf<unsigned char> raw_in;
    DevBuf<unsigned char> raw_out;
};

// Dithered integer output (r8bgpu_batch_set_dither), created by the first setting: the channels' settings on both sides,
// their error histories ([n_ch][16], e[j] at slot j & 15), and the per-call records of k_dither_shape, uploaded from two
// alternating pinned buffers.
static_assert(sizeof(DitherCfg) == sizeof(r8bgpu_dither) && offsetof(DitherCfg, taps) == offsetof(r8bgpu_dither, taps),
              "DitherCfg mirrors r8bgpu_dither");
struct DitherState {
    std::vector<DitherCfg> cfg;
    bool any = false; // some channel is not OFF
    DevBuf<DitherCfg> d_cfg;
    DevBuf<double> d_err;
    RecRing<DitherRec> rec;
    std::vector<long long> m; // per channel: dithered outputs since its clear (the history ring's index)
    DevBuf<DitherCall> d_call; // {d_cfg, rec.d, d_err}, for the fused kernel's stores
    DevBuf<double> d_zero;     // zeros: the fp64 tail of a passthrough part's flush
};

// Moving streams (r8bgpu_batch_export / _import): scratch of the calls that move state blobs, created by the first one.
struct StateStaging {
    DevBuf<unsigned char> d_blob; // device blobs of the host forms
    PinBuf<unsigned char> h_blob; // pinned host blobs of the host forms
    DevBuf<unsigned char> d_aux;  // segment records, header words, checksums
};

// Long clips (r8bgpu_batch_oneshot / _oneshot_host), created by the first one: the per-call lane records ([2][lane]:
// gather, scatter) and, for the host form, the pinned blocks the lanes' samples cross PCIe in; h2d is recorded after each
// upload of h_in, which is refilled only once that upload has run.
struct OneshotStaging {
    RecRing<OneshotRec> rec;
    PinBuf<unsigned char> h_in, h_out;
    Event h2d;
};

// One-bit DSD output (r8bgpu_batch_set_dsd_out), present while it is on: each channel's modulator state on the device and
// its count of held-back bits on the host, the per-call records of k_dsd_mod (two alternating pinned buffers), the fp64
// rows the resampler writes for the modulator, and for the host forms the device blocks of the caller's input bytes and
// of the output bytes as they cross PCIe.
struct DsdOutState {
    DevBuf<DsdModState> d_state;
    std::vector<int> pend;
    RecRing<DsdModRec> rec;
    DevBuf<double> d_y;
    size_t y_cap = 0; // samples per row
    DevBuf<unsigned char> d_in;
    DevBuf<unsigned char> d_bytes;
};

struct r8bgpu_batch {
    // The first members, so destroyed last: the destructor makes the batch's device current here, so that every owner
    // below releases its memory, events and streams with that device current; dev_bytes is what they charge.
    std::optional<DeviceGuard> releasing;
    unsigned long long dev_bytes = 0;
    std::unique_ptr<DsdOutState> dsd; // ordinary and mixed batches: non-null while DSD output is on (a front's shards own theirs)
    std::unique_ptr<StateStaging> stx; // ordinary and mixed batches: null until a stream is exported or imported
    std::unique_ptr<OneshotStaging> osx; // ordinary batches: null until the first long-clip call
    std::unique_ptr<DitherState> dith; // ordinary and mixed batches: null until a channel is set (a front's shards own theirs)
    std::unique_ptr<ShardFront> front; // non-null: multi-device front (everything below except plan/n_ch is unused)
    std::unique_ptr<MixedFront> mixed; // non-null: mixed batch (device, stream, launches and dev_bytes are its own)
    const Plan* plan = nullptr;
    Plan plan_copy; // batches own a copy so the plan handle may be destroyed first
    int n_ch = 0;
    int device = 0;
    cudaStream_t stream = nullptr;
    Schedule sched; // every channel's schedule while they run in lock-step
    bool diverged = false; // channels' schedules differ (ragged calls, clear_channels): rag holds them
    RaggedSchedule rag;
    // ragged launches: per-channel records [slot][channel] (slots 0..ns-1: link-ring refill, ns..2ns: the call's stages and
    // the history copy), uploaded from two alternating pinned buffers; links_fresh: the rings of stages that lock-step
    // calls fuse away hold the streams' recent past
    RecRing<RaggedRec> rec;
    bool links_fresh = false;
    std::vector<StageDev> dev;
    std::vector<StageCall> calls;
    unsigned long long launches = 0;
    // optional per-stage device timing (CUDA events on the launch stream)
    bool timing = false;
    struct EvPair {
        int stage;
        Event a, b;
    };
    std::vector<EvPair> events;
    std::vector<double> stage_ms;
    std::vector<unsigned long long> stage_launches;
    // staging + pipeline resources for the host-pointer entry point
    DevBuf<double> st_in;
    DevBuf<double> st_out;
    DevBuf<unsigned char> raw_in; // narrow-format staging (r8b_format.cu)
    DevBuf<unsigned char> raw_out;
    // flushes (r8bgpu_batch_flush / _flush_host): fp64 output block and typed output block, fl_cap samples per channel
    DevBuf<double> fl_out;
    DevBuf<unsigned char> fl_raw;
    size_t fl_cap = 0;
    std::vector<long long> pass_n; // passthrough plans (no stages, no schedule totals): input samples since clear, per channel
    std::vector<double> trim;      // trim plans: each channel's factor (r8bgpu_batch_set_trim); empty otherwise
    Stream s_h2d, s_d2h, s_comp;
    int host_groups = 1;
    std::vector<Event> ev_h2d, ev_k;
    DevBuf<unsigned long long> prof; // R8BGPU_PROFILE: phase cycle counters of the fused kernel
    int n_sm = 0;     // SMs of the device (grid of the persistent v2 fused kernel)
    int f2_flags = 6; // v2 fused kernel: bit 0 ping-pong token, bit 1 bulk-copied input tiles, bit 2 interpolation on the fp64 tensor path
    bool f2_flags_env = false; // R8BGPU_F2_FLAGS set: its flags are used as given
    unsigned long long prof_ctas = 0;
    bool prof_v2 = false; // the counters hold k_up2_frac2's per-tile phases (slots 0-8), prof_ctas counts tiles

    ~r8bgpu_batch()
    {
        if (front) { // its workers stop before its shards go
            front->pool.reset();
            return;
        }
        releasing.emplace(device);
        if (mixed) { // the parts' queued work ends before the parts go, and the parts before the streams they borrow
            cudaStreamSynchronize(stream);
            mixed->parts.clear();
        }
        unsigned long long h[10] = {};
        if (prof != nullptr && cudaDeviceSynchronize() == cudaSuccess &&
            cudaMemcpy(h, prof, sizeof h, cudaMemcpyDeviceToHost) == cudaSuccess) {
            if (prof_v2) {
                // slots: see k_up2_frac2; 5 = E time summed over the 8 warps of a half, 6 = the slowest warp's, 8 + 7 = E
                const double n = prof_ctas ? (double) prof_ctas : 1.0;
                const unsigned long long tot = h[0] + h[1] + h[2] + h[3] + h[4] + h[7] + h[8];
                auto line = [&](const char* nm, double v) {
                    fprintf(stderr, "  %-26s %9.0f  (%4.1f %%)\n", nm, v / n, tot ? 100.0 * v / tot : 0.0);
                };
                fprintf(stderr, "[r8bgpu profile] k_up2_frac2 phases, mean clk per tile (one half-CTA) over %llu tiles:\n", prof_ctas);
                line("A_wait landed tile", (double) h[0]);
                line("A_work gather+fwd1", (double) h[1]);
                line("A_bar", (double) h[2]);
                line("B fwd2+fwd3", (double) h[3]);
                line("C+D split*G, inverse", (double) h[4]);
                line("E interp", (double) (h[7] + h[8]));
                line("  E_work mean over warps", h[5] / 8.0);
                line("  E_work max over warps", (double) h[6]);
                line("  E_bar (thread 0)", (double) h[7]);
                fprintf(stderr, "  %-26s %9.0f\n", "total", tot / n);
            } else {
                static const char* nm[8] = {"gather+fwd1", "fwd2", "fwd3", "C(split*G)", "inv1", "inv2", "inv3+ystore", "interp"};
                unsigned long long tot = 0;
                for (int i = 0; i < 8; i++) tot += h[i];
                fprintf(stderr, "[r8bgpu profile] k_up2_frac phases, mean clk per CTA over %llu CTAs:\n", prof_ctas);
                for (int i = 0; i < 8; i++)
                    fprintf(stderr, "  %-12s %9.0f  (%4.1f %%)\n", nm[i], prof_ctas ? (double) h[i] / prof_ctas : 0.0,
                            tot ? 100.0 * h[i] / tot : 0.0);
                if (h[8] + h[9] > 0)
                    fprintf(stderr, "  order-2 bank, clk per CTA: 4-output groups %.0f, queued single outputs %.0f\n",
                            (double) h[8] / prof_ctas, (double) h[9] / prof_ctas);
            }
        }
    }
};

// ---- per-channel calls: which batch runs a channel, and the caller's channel list -------------------------------------

// The batches a front (shards) or a mixed batch (parts) is made of; none for an ordinary batch.
static const std::vector<std::unique_ptr<r8bgpu_batch>>* sub_batches(const r8bgpu_batch* b)
{
    return b->front ? &b->front->shards : b->mixed ? &b->mixed->parts : nullptr;
}

// The single-plan batches b is made of: its shards or parts, else b itself.
static std::vector<const r8bgpu_batch*> plan_batches(const r8bgpu_batch* b)
{
    const auto* subs = sub_batches(b);
    if (subs == nullptr) return {b};
    std::vector<const r8bgpu_batch*> v;
    for (const auto& sb : *subs) v.push_back(sb.get());
    return v;
}

// Where channel c of a batch runs: row `row` of batch b, which is sub-batch `sub` of a front (its shard) or of a mixed
// batch (its part), or the batch itself (sub 0).
struct Slot {
    r8bgpu_batch* b;
    int row, sub;
};

static Slot slot_of(const r8bgpu_batch* b, int c)
{
    if (b->front) { // the last shard whose first channel is at most c
        const std::vector<int>& ch0 = b->front->ch0;
        const int s = (int) (std::upper_bound(ch0.begin(), ch0.end(), c) - ch0.begin()) - 1;
        return Slot{b->front->shards[(size_t) s].get(), c - ch0[(size_t) s], s};
    }
    if (b->mixed) {
        const int p = b->mixed->part_of[(size_t) c];
        return Slot{b->mixed->parts[(size_t) p].get(), b->mixed->row_of[(size_t) c], p};
    }
    return Slot{const_cast<r8bgpu_batch*>(b), c, 0};
}

// A caller's channel list grouped by the batch that runs each channel: one group per shard or part (empty where no
// channel falls), one for an ordinary batch.  rows: the channels' rows there; idx: their positions in the caller's list;
// both in the caller's order.
struct ChannelGroup {
    r8bgpu_batch* b;
    std::vector<int> rows, idx;
};

static std::vector<ChannelGroup> group_channels(const r8bgpu_batch* b, const int* channels, int n)
{
    const auto* subs = sub_batches(b);
    std::vector<ChannelGroup> g(subs ? subs->size() : 1);
    for (size_t k = 0; k < g.size(); k++) g[k].b = subs ? (*subs)[k].get() : const_cast<r8bgpu_batch*>(b);
    for (int i = 0; i < n; i++) {
        const Slot s = slot_of(b, channels[i]);
        g[(size_t) s.sub].rows.push_back(s.row);
        g[(size_t) s.sub].idx.push_back(i);
    }
    return g;
}

// A per-channel payload of the caller (v[i] for position i of its list) for the positions idx of a group.
template <class T>
static std::vector<T> gather(const T* v, const std::vector<int>& idx)
{
    std::vector<T> out;
    out.reserve(idx.size());
    for (int i : idx) out.push_back(v[i]);
    return out;
}

// Refuses a caller's channel list that names an index out of range or, when `distinct`, a channel twice (in the caller's
// numbers).  each(i, c) runs the call's own checks of channel c = channels[i] in the same pass, so that a list with
// several faults reports the first of them.
static bool check_channels(const r8bgpu_batch* b, const int* channels, int n, const char* what, bool distinct,
                           const std::function<bool(int, int)>& each = nullptr)
{
    std::vector<char> named(distinct ? (size_t) b->n_ch : 0, 0);
    for (int i = 0; i < n; i++) {
        const int c = channels[i];
        if (c < 0 || c >= b->n_ch) {
            set_err(std::string(what) + ": channel index out of range");
            return false;
        }
        if (distinct) {
            if (named[(size_t) c]) {
                set_err(std::string(what) + ": channel " + std::to_string(c) + " named twice");
                return false;
            }
            named[(size_t) c] = 1;
        }
        if (each && !each(i, c)) return false;
    }
    return true;
}

// DSD output is on (r8bgpu_batch_set_dsd_out): a front asks its shards, which all share the setting.
static bool dsd_on(const r8bgpu_batch* b)
{
    return b != nullptr && (b->front ? b->front->shards[0]->dsd != nullptr : b->dsd != nullptr);
}

// Bits a call may return for up to `bound` resampler outputs after up to 7 held-back bits, whole bytes only; a flush
// also fills its last byte with silence.
static int dsd_out_bound(long long bound) { return (int) ((bound + 7) / 8 * 8); }
static int dsd_flush_bound(long long bound) { return (int) ((bound + 14) / 8 * 8); }

// While DSD output is on, the calls whose output is fp64 by signature are refused.
static bool refuse_dsd_plain(const r8bgpu_batch* b, const char* what)
{
    if (!dsd_on(b)) return false;
    set_err(std::string(what) + ": DSD output is on (r8bgpu_batch_set_dsd_out): the output must be R8BGPU_DSD_LSB or "
            "R8BGPU_DSD_MSB (use the _fmt calls)");
    return true;
}

// The named channels' modulators restart (stream order on st); channels == nullptr: every channel.
static bool dsd_clear(r8bgpu_batch* b, const int* channels, int n, cudaStream_t st)
{
    if (!b->dsd) return true;
    DsdOutState& D = *b->dsd;
    if (channels == nullptr) {
        std::fill(D.pend.begin(), D.pend.end(), 0);
        return cuda_ok(cudaMemsetAsync(D.d_state, 0, (size_t) b->n_ch * sizeof(DsdModState), st), "dsd: clear");
    }
    for (int i = 0; i < n; i++) {
        D.pend[(size_t) channels[i]] = 0;
        if (!cuda_ok(cudaMemsetAsync(D.d_state + channels[i], 0, sizeof(DsdModState), st), "dsd: clear")) return false;
    }
    return true;
}

// Channel c's input and output totals since its clear.
static void channel_totals_of(const r8bgpu_batch* b, int c, long long& n_in, long long& n_out)
{
    const Slot s = slot_of(b, c);
    if (s.b->plan->passthrough) {
        n_in = n_out = s.b->pass_n[(size_t) s.row];
        return;
    }
    const Schedule& S = s.b->diverged ? s.b->rag.of(s.row) : s.b->sched;
    n_in = S.inputs();
    n_out = S.outputs();
}

// Each channel's output total before a call: the index at which a dithered channel's noise sequence continues.
static std::vector<long long> outputs_before(const r8bgpu_batch* b)
{
    std::vector<long long> n0((size_t) b->n_ch);
    long long n_in = 0;
    for (int c = 0; c < b->n_ch; c++) channel_totals_of(b, c, n_in, n0[(size_t) c]);
    return n0;
}

// ---- dithered integer output: the pieces every call path shares ----------------------------------------------------

static bool dither_cfg_ok(const r8bgpu_dither& d, std::string& why)
{
    if (d.kind != R8BGPU_DITHER_OFF && d.kind != R8BGPU_DITHER_TPDF) {
        why = "unknown kind " + std::to_string(d.kind);
        return false;
    }
    if (d.n_taps < 0 || d.n_taps > R8BGPU_DITHER_MAX_TAPS) {
        why = "n_taps " + std::to_string(d.n_taps) + " outside 0.." + std::to_string(R8BGPU_DITHER_MAX_TAPS);
        return false;
    }
    if (d.kind == R8BGPU_DITHER_OFF && d.n_taps > 0) {
        why = "taps with kind OFF";
        return false;
    }
    for (int k = 0; k < d.n_taps; k++)
        if (!std::isfinite(d.taps[k])) {
            why = "tap " + std::to_string(k + 1) + " is not finite";
            return false;
        }
    return true;
}

// the formats a dither applies to: U8 quantises to int8, µ-law / A-law to the int16 value they encode (dither_range)
static bool is_int_format(int fmt) { return fmt == FMT_S16 || fmt == FMT_S24 || fmt == FMT_S32 || is_byte_format(fmt); }

// A call writing `fmt` into channels [ch0, ch0 + nch) of b has a dithered channel.
static bool dither_active(const r8bgpu_batch* b, int fmt, int ch0, int nch)
{
    if (!b->dith || !b->dith->any || !is_int_format(fmt)) return false;
    for (int c = ch0; c < ch0 + nch; c++)
        if (b->dith->cfg[(size_t) c].kind != R8BGPU_DITHER_OFF) return true;
    return false;
}

// This call's host records (their previous upload has finished); the caller fills the channels it converts.
static DitherRec* dither_records(r8bgpu_batch* b)
{
    DitherState& D = *b->dith;
    return D.rec.next("dither: records");
}

// Some dithered channel among [ch0, ch0 + nch) has taps (such a call cannot dither in the fused kernel's stores).
static bool dither_shaped(const r8bgpu_batch* b, int ch0, int nch)
{
    for (int c = ch0; c < ch0 + nch; c++) {
        const DitherCfg& d = b->dith->cfg[(size_t) c];
        if (d.kind != R8BGPU_DITHER_OFF && d.n_taps > 0) return true;
    }
    return false;
}

// Completes the records of channels [ch0, ch0 + nch) (the caller set row, n, n0) with each channel's history index and
// uploads them; the dithered channels' counts advance.  max_flat / max_shaped: the largest count of either kind.
static bool dither_upload(r8bgpu_batch* b, int ch0, int nch, cudaStream_t st, long long& max_flat, long long& max_shaped)
{
    DitherState& D = *b->dith;
    DitherRec* h = D.rec.host() + ch0;
    max_flat = max_shaped = 0;
    for (int c = 0; c < nch; c++) {
        const DitherCfg& d = D.cfg[(size_t) (ch0 + c)];
        long long& m = D.m[(size_t) (ch0 + c)];
        h[c].m0 = m;
        if (d.kind == R8BGPU_DITHER_OFF || h[c].n <= 0) continue;
        m += h[c].n;
        (d.n_taps > 0 ? max_shaped : max_flat) = std::max(d.n_taps > 0 ? max_shaped : max_flat, h[c].n);
    }
    if (max_flat + max_shaped == 0) return true;
    return D.rec.upload((size_t) ch0, (size_t) nch, st, "dither: record upload");
}

// Re-quantises the dithered channels among [ch0, ch0 + nch) of `out` (a device buffer that the usual conversion has
// filled; out's channel 0 is b's channel ch0) from the fp64 rows of this call's records: one launch for the flat channels
// (frames split over CTAs), one for the shaped ones (one pass each).
static bool dither_launch(r8bgpu_batch* b, const r8bgpu_buffer& out, int ch0, int nch, cudaStream_t st)
{
    DitherState& D = *b->dith;
    long long max_flat = 0, max_shaped = 0;
    if (!dither_upload(b, ch0, nch, st, max_flat, max_shaped)) return false;
    for (int shaped = 0; shaped < 2; shaped++) {
        const long long max_n = shaped ? max_shaped : max_flat;
        if (max_n == 0) continue;
        launch_dither(out.format, out.data, out.interleaved != 0, out.stride, D.rec.d + ch0, D.d_cfg + ch0,
                      D.d_err + (size_t) ch0 * kDitherTaps, (int) max_n, nch, out.scale, shaped != 0, st);
        b->launches++;
    }
    return true;
}

// The named channels' error histories restart (stream order on st).
static bool dither_clear(r8bgpu_batch* b, const int* channels, int n, cudaStream_t st)
{
    if (!b->dith) return true;
    for (int i = 0; i < n; i++) b->dith->m[(size_t) channels[i]] = 0;
    for (int i = 0; i < n; i++)
        if (!cuda_ok(cudaMemsetAsync(b->dith->d_err + (size_t) channels[i] * kDitherTaps, 0, kDitherTaps * sizeof(double), st),
                     "dither: clear"))
            return false;
    return true;
}

static bool dither_clear_all(r8bgpu_batch* b, cudaStream_t st)
{
    if (!b->dith) return true;
    std::fill(b->dith->m.begin(), b->dith->m.end(), 0LL);
    return cuda_ok(cudaMemsetAsync(b->dith->d_err, 0, (size_t) b->n_ch * kDitherTaps * sizeof(double), st), "dither: clear");
}

extern "C" {

const char* r8bgpu_last_error(void) { return g_err.c_str(); }
const char* r8bgpu_version(void) { return "r8bgpu 0.1 (sm_90a)"; }

r8bgpu_plan* r8bgpu_plan_create(double src, double dst, int max_in_len, double tb, double atten, int phase,
                                int extfft, int fasttiming)
{
    std::unique_ptr<r8bgpu_plan> h(new r8bgpu_plan);
    if (!h->p.build(src, dst, max_in_len, tb, atten, phase, extfft, fasttiming)) {
        set_err("plan_create: " + h->p.error);
        return nullptr;
    }
    return h.release();
}

r8bgpu_plan* r8bgpu_plan_create_trim(double src, double dst, int max_in_len, double tb, double atten, int extfft,
                                     double max_trim)
{
    std::unique_ptr<r8bgpu_plan> h(new r8bgpu_plan);
    if (!h->p.build_trim(src, dst, max_in_len, tb, atten, extfft, max_trim)) {
        set_err("plan_create_trim: " + h->p.error);
        return nullptr;
    }
    return h.release();
}

r8bgpu_plan* r8bgpu_plan_create_asrc(double src, double dst, int max_in_len, double tb, double atten, int extfft,
                                     double max_trim)
{
    std::unique_ptr<r8bgpu_plan> h(new r8bgpu_plan);
    if (!h->p.build_trim(src, dst, max_in_len, tb, atten, extfft, max_trim, true)) {
        set_err("plan_create_asrc: " + h->p.error);
        return nullptr;
    }
    return h.release();
}

double r8bgpu_plan_max_trim(const r8bgpu_plan* plan) { return plan->p.max_trim; }

int r8bgpu_plan_simulate_trim(const r8bgpu_plan* plan, int n_calls, const int* lens, const double* factors, int* counts,
                              long long* next_pos, double* next_frac)
{
    const Plan& P = plan->p;
    if (P.trim_stage < 0) {
        set_err("simulate_trim: not a trim plan (r8bgpu_plan_create_trim)");
        return -1;
    }
    if (n_calls < 0 || (n_calls > 0 && (lens == nullptr || factors == nullptr || counts == nullptr))) {
        set_err("simulate_trim: bad arguments");
        return -1;
    }
    for (int i = 0; i < n_calls; i++) {
        if (lens[i] < 0 || lens[i] > P.max_in_len) {
            set_err("simulate_trim: block length outside [0, MaxInLen]");
            return -1;
        }
        if (!P.trim_factor_ok(factors[i])) {
            set_err("simulate_trim: factor outside [1 - max_trim, 1 + max_trim]");
            return -1;
        }
    }
    // one channel through the batch's own host code: the factor's re-base, then the call
    Schedule sc;
    sc.init(&P);
    RaggedSchedule rs;
    rs.init(sc, 1);
    RaggedSchedule::Step step;
    const int ch = 0;
    for (int i = 0; i < n_calls; i++) {
        const double dsr = P.trim_dsr(factors[i]);
        rs.retime_channels(&ch, 1, &dsr);
        rs.plan_call(lens + i, step);
        counts[i] = step.count[0];
        rs.commit(step);
        const Schedule::PolyState& ps = rs.groups[0].poly[(size_t) P.trim_stage];
        if (next_pos != nullptr) next_pos[i] = ps.p;
        if (next_frac != nullptr) next_frac[i] = ps.fpos;
    }
    return 0;
}

r8bgpu_plan* r8bgpu_plan_create_stage(int kind, const double* params, int n_params, int max_in_len, int extfft)
{
    double a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < n_params && i < 8; i++) a[i] = params[i];
    std::unique_ptr<r8bgpu_plan> h(new r8bgpu_plan);
    if (max_in_len <= 0 || !h->p.build_single(kind, a, max_in_len, extfft)) {
        set_err("plan_create_stage: " + h->p.error);
        return nullptr;
    }
    return h.release();
}

void r8bgpu_plan_destroy(r8bgpu_plan* plan) { delete plan; }
int r8bgpu_plan_max_out_len(const r8bgpu_plan* plan) { return plan->p.max_out_len; }
int r8bgpu_plan_in_len_before_out_pos(const r8bgpu_plan* plan, int pos) { return plan->p.in_len_before_out_pos(pos); }
int r8bgpu_plan_input_required_for_output(const r8bgpu_plan* plan, int n) { return plan->p.input_required_for_output(n); }
double r8bgpu_plan_latency_frac(const r8bgpu_plan*) { return 0.0; } // linear-phase chains leave no fractional latency
int r8bgpu_plan_is_passthrough(const r8bgpu_plan* plan) { return plan->p.passthrough ? 1 : 0; }
int r8bgpu_plan_stage_count(const r8bgpu_plan* plan) { return (int) plan->p.stages.size(); }

static int stage_data_len(const StageDesc& s)
{
    switch (s.kind) {
    case ST_BLOCKCONV: return s.lp.kernel_len;
    case ST_FRAC_WHOLE:
    case ST_FRAC_POLY: return (int) s.bank.table.size();
    default: return s.hb_taps;
    }
}

int r8bgpu_plan_stage_info(const r8bgpu_plan* plan, int stage, r8bgpu_stage_info* info)
{
    if (stage < 0 || stage >= (int) plan->p.stages.size() || info == nullptr) {
        set_err("stage_info: bad stage index");
        return -1;
    }
    const StageDesc& s = plan->p.stages[(size_t) stage];
    memset(info, 0, sizeof *info);
    info->kind = (int) s.kind;
    info->up = s.up;
    info->down = s.down;
    info->max_out_len = s.max_out_len;
    info->data_len = stage_data_len(s);
    switch (s.kind) {
    case ST_BLOCKCONV:
        info->kernel_len = s.lp.kernel_len;
        info->latency = s.latency;
        info->ref_input_len = s.ref_input_len;
        info->block_len_bits = s.lp.block_len_bits;
        break;
    case ST_FRAC_WHOLE:
    case ST_FRAC_POLY:
        info->kernel_len = s.bank.filter_len;
        info->fracs = s.bank.fracs;
        info->in_step = s.in_step;
        info->out_step = s.out_step;
        info->order = s.bank.order;
        info->atten = s.bank.atten;
        break;
    default:
        info->kernel_len = s.hb_taps;
        info->atten = s.hb_atten;
        break;
    }
    return 0;
}

int r8bgpu_plan_stage_data(const r8bgpu_plan* plan, int stage, double* out, int cap)
{
    if (stage < 0 || stage >= (int) plan->p.stages.size()) {
        set_err("stage_data: bad stage index");
        return -1;
    }
    const StageDesc& s = plan->p.stages[(size_t) stage];
    const double* src = s.kind == ST_BLOCKCONV ? s.lp.taps.data()
        : (s.kind == ST_FRAC_WHOLE || s.kind == ST_FRAC_POLY) ? s.bank.table.data() : s.hb.data();
    const int n = stage_data_len(s);
    const int c = n < cap ? n : cap;
    if (out != nullptr && c > 0) memcpy(out, src, (size_t) c * sizeof(double));
    return n;
}

int r8bgpu_plan_describe(const r8bgpu_plan* plan, char* buf, int cap)
{
    const std::string d = plan->p.describe();
    if (buf != nullptr && cap > 0) {
        const size_t n = d.size() < (size_t) cap - 1 ? d.size() : (size_t) cap - 1;
        memcpy(buf, d.data(), n);
        buf[n] = 0;
    }
    return (int) d.size();
}

int r8bgpu_plan_simulate(const r8bgpu_plan* plan, const int* lens, int n_calls, int* counts)
{
    Schedule sc;
    sc.init(&plan->p);
    std::vector<StageCall> calls;
    for (int i = 0; i < n_calls; i++) {
        if (lens[i] < 0 || lens[i] > plan->p.max_in_len) {
            set_err("simulate: block length outside [0, MaxInLen]");
            return -1;
        }
        counts[i] = sc.advance(lens[i], calls);
    }
    return 0;
}

int r8bgpu_plan_fused_info(const r8bgpu_plan* plan, int stage, r8bgpu_fused_info* info)
{
    const auto& st = plan->p.stages;
    if (stage < 0 || stage >= (int) st.size() || info == nullptr || st[(size_t) stage].kind != ST_BLOCKCONV) {
        set_err("plan_fused_info: stage is not a BlockConvolver stage of the plan");
        return -1;
    }
    const FusedPlan fp = plan_fused_stage(st, (size_t) stage, fused_knobs_env());
    memset(info, 0, sizeof *info);
    info->kernel = fp.kernel;
    info->up = fp.geom.ok ? fp.geom.up : fp.copy ? 2 : 0;
    info->copy = fp.copy;
    info->ysh = fp.geom.ok ? fp.geom.ysh : 31;
    info->pad = info->ysh != 31;
    info->cs = fp.cs;
    if (fp.whole) {
        const StageDesc& f = st[(size_t) stage + 1];
        info->in_step = f.in_step;
        info->out_step = f.out_step;
        info->tc_n_groups = fp.tc.n_groups;
        info->tc_smaxp = fp.tc.smaxp;
        info->ir = fp.fma.ir;
        info->fma_n_groups = fp.fma.n_groups;
        info->fma_smaxp = fp.fma.smaxp;
        info->tc_fits = fp.tc_fits;
        info->fma_fits = fp.fma_fits;
        info->bank_in_smem = fp.bank_in_smem;
    }
    return 0;
}

int r8bgpu_plan_cascade_info(const r8bgpu_plan* plan, int stage, r8bgpu_hb_info* info)
{
    const auto& st = plan->p.stages;
    if (stage < 0 || stage >= (int) st.size() || info == nullptr ||
        (st[(size_t) stage].kind != ST_HBUP && st[(size_t) stage].kind != ST_HBDOWN)) {
        set_err("plan_cascade_info: stage is not a half-band stage of the plan");
        return -1;
    }
    // walk the runs as r8bgpu_batch_create does (no earlier kernel covers a run's first half-band stage)
    const HbKnobs k = hb_knobs_env();
    size_t i = 0;
    HbRunPlan hr;
    for (;;) {
        while (st[i].kind != ST_HBUP && st[i].kind != ST_HBDOWN) i++;
        hr = plan_hb_run(st, i, k);
        if ((int) i + hr.n_stages > stage) break;
        i += (size_t) hr.n_stages;
    }
    memset(info, 0, sizeof *info);
    info->first = (int) i;
    if ((int) i < stage) {
        info->kind = R8BGPU_HB_INSIDE;
        return 0;
    }
    const int c = hr.n_stages;
    const bool up = st[i].kind == ST_HBUP;
    info->kind = c < 2 ? R8BGPU_HB_SINGLE : up ? R8BGPU_HB_UP_CASCADE : R8BGPU_HB_DOWN_CASCADE;
    info->n_stages = c;
    for (int s = 0; s < c; s++) info->ntaps[s] = st[i + (size_t) s].hb_taps;
    info->writes_ring = i + (size_t) c < st.size();
    if (c < 2) return 0;
    info->smem_bytes = hr.smem_bytes;
    if (up) {
        info->fuse_last2 = hr.up.fuse_last2;
        info->n_buffers = c - hr.up.fuse_last2;
        info->w = hr.up.w;
        for (int s = 0; s <= c; s++) {
            info->lo_off[s] = hr.up.lo_off[s];
            info->hi_off[s] = hr.up.hi_off[s];
        }
    } else {
        info->n_buffers = c;
        info->w = hr.down.w;
        for (int s = 0; s <= c; s++) info->back[s] = hr.down.back[s];
    }
    return 0;
}

int r8bgpu_plan_blockconv_info(const r8bgpu_plan* plan, int stage, int n_channels, r8bgpu_blockconv_info* info)
{
    const auto& st = plan->p.stages;
    if (stage < 0 || stage >= (int) st.size() || info == nullptr || st[(size_t) stage].kind != ST_BLOCKCONV ||
        n_channels <= 0 || n_channels > 65535) {
        set_err("plan_blockconv_info: need a BlockConvolver stage of the plan and 1..65535 channels");
        return -1;
    }
    const StageDesc& s = st[(size_t) stage];
    const BcPlan bp = plan_blockconv_stage(s, plan_fused_stage(st, (size_t) stage, fused_knobs_env()), n_channels,
                                           bcl_scratch_cap_env());
    if (!bp.err.empty()) {
        set_err("plan_blockconv_info: " + bp.err);
        return -1;
    }
    memset(info, 0, sizeof *info);
    info->kernel = bp.kernel;
    info->fft_log2 = bp.t.fft_log2;
    info->up = bp.t.up;
    info->src_up = bp.t.virt_up;
    info->down = s.down;
    info->block_exact = s.block_exact;
    info->trunc = bp.trunc;
    info->nyq_bin = bp.trunc > 0 ? (1 << bp.t.fft_log2) / (2 * bp.trunc) : 0;
    info->lg = bp.t.lg;
    info->adv = bp.adv;
    info->smem_bytes = bp.smem_bytes;
    if (bp.t.large) {
        info->r0 = 1 << (bp.t.fft_log2 - 12);
        info->scratch_tiles = bp.scratch_tiles;
        info->scratch_bytes_per_ch = bp.scratch_per_ch;
        info->group_ch = bp.group_ch;
    }
    return 0;
}

int r8bgpu_plan_frac_info(const r8bgpu_plan* plan, int stage, r8bgpu_frac_info* info)
{
    const auto& st = plan->p.stages;
    if (stage < 0 || stage >= (int) st.size() || info == nullptr ||
        (st[(size_t) stage].kind != ST_FRAC_WHOLE && st[(size_t) stage].kind != ST_FRAC_POLY)) {
        set_err("plan_frac_info: stage is not an interpolator stage of the plan");
        return -1;
    }
    const StageDesc& s = st[(size_t) stage];
    const FracPlan f = plan_frac_stage(plan->p, (size_t) stage);
    if (!f.err.empty()) {
        set_err("plan_frac_info: " + f.err);
        return -1;
    }
    memset(info, 0, sizeof *info);
    const bool fused = stage > 0 && plan_fused_stage(st, (size_t) stage - 1, fused_knobs_env()).geom.ok;
    info->kernel = fused ? R8BGPU_FRAC_FUSED : s.kind == ST_FRAC_WHOLE ? R8BGPU_FRAC_WHOLE : R8BGPU_FRAC_POLY;
    info->flen = s.bank.filter_len;
    info->fll = s.bank.filter_len / 2 - 1;
    info->fracs = s.kind == ST_FRAC_POLY ? s.bank.fracs : 0;
    info->tile = f.tile;
    info->window = frac_window(f.tile, f.in_per_out, info->flen);
    info->tile_ragged = f.tile_ragged;
    info->window_ragged = frac_window(f.tile_ragged, f.in_per_out_ragged, info->flen);
    info->frac_cap = FRAC_CAP;
    return 0;
}

int r8bgpu_plan_order2_info(const r8bgpu_plan* plan, int stage, double trim_factor, int span, r8bgpu_order2_info* info)
{
    const Plan& P = plan->p;
    const auto& st = P.stages;
    if (stage < 0 || stage + 1 >= (int) st.size() || info == nullptr || st[(size_t) stage + 1].kind != ST_FRAC_POLY) {
        set_err("plan_order2_info: stage is not a BlockConvolver fused with an order-2 interpolator");
        return -1;
    }
    const FusedPlan fp = plan_fused_stage(st, (size_t) stage, fused_knobs_env());
    if (fp.kernel != R8BGPU_FUSED_ORDER2) {
        set_err("plan_order2_info: stage is not a BlockConvolver fused with an order-2 interpolator");
        return -1;
    }
    if (trim_factor != 1.0 && ((int) stage + 1 != P.trim_stage || !P.trim_factor_ok(trim_factor))) {
        set_err("plan_order2_info: a factor other than 1 needs a trim plan and must lie in [1 - max_trim, 1 + max_trim]");
        return -1;
    }
    if (span < 0) {
        set_err("plan_order2_info: span must be >= 0");
        return -1;
    }
    const StageDesc& f = st[(size_t) stage + 1];
    const double dsr = (int) stage + 1 == P.trim_stage ? P.trim_dsr(trim_factor) : f.dst_rate;
    const long long range = span > 0 ? span : 2LL * fp.geom.span_max;
    const PolyCall pc = plan_poly_call(f, fp.geom, fp.poly_v2, f.src_rate, dsr, 0, range, -1, poly_knobs_env());
    memset(info, 0, sizeof *info);
    info->poly_v2 = pc.v2;
    info->n_tiles = pc.n_tiles;
    info->span = pc.span;
    info->span_max = fp.geom.span_max;
    info->poly_dir = pc.poly_dir;
    info->poly_rows_cap = pc.poly_rows_cap;
    info->poly_row_stride = pc.poly_row_stride;
    info->poly_chunks = pc.poly_chunks;
    info->poly_n = pc.poly_n;
    info->ysh = pc.ysh;
    info->smem_bytes = pc.smem_bytes;
    info->flen = f.bank.filter_len;
    info->fracs = f.bank.fracs;
    info->ratio = f.src_rate / dsr;
    return 0;
}

int r8bgpu_plan_simulate_ragged(const r8bgpu_plan* plan, int n_channels, int n_calls, const int* lens, const int* clear,
                                int* counts, int* groups)
{
    if (n_channels <= 0 || n_calls < 0 || lens == nullptr || counts == nullptr) {
        set_err("simulate_ragged: bad arguments");
        return -1;
    }
    Schedule sc;
    sc.init(&plan->p);
    RaggedSchedule rs;
    rs.init(sc, n_channels);
    RaggedSchedule::Step step;
    std::vector<int> named;
    for (int i = 0; i < n_calls; i++) {
        const int* li = lens + (size_t) i * n_channels;
        for (int c = 0; c < n_channels; c++)
            if (li[c] < 0 || li[c] > plan->p.max_in_len) {
                set_err("simulate_ragged: block length outside [0, MaxInLen]");
                return -1;
            }
        if (clear != nullptr) {
            named.clear();
            for (int c = 0; c < n_channels; c++)
                if (clear[(size_t) i * n_channels + c]) named.push_back(c);
            rs.clear_channels(named.data(), (int) named.size());
        }
        rs.plan_call(li, step);
        for (int c = 0; c < n_channels; c++) counts[(size_t) i * n_channels + c] = step.count[(size_t) step.key_of[(size_t) c]];
        rs.commit(step);
        if (groups != nullptr) groups[i] = (int) rs.groups.size();
    }
    return 0;
}

static const char* kTrimDefaultFlush =
    "a trim plan has no default flush target (ceil(N * dst / src) means nothing once the ratio has moved); pass explicit "
    "targets (absolute output counts, see r8bgpu_batch_channel_totals)";

int r8bgpu_plan_flush_max_out_len(const r8bgpu_plan* plan)
{
    if (plan->p.trim_stage >= 0) {
        set_err(std::string("plan_flush_max_out_len: ") + kTrimDefaultFlush);
        return -1;
    }
    return flush_max_out_len(plan->p);
}

int r8bgpu_plan_simulate_flush(const r8bgpu_plan* plan, int n_calls, const int* lens, long long target, long long* zeros_fed,
                               int* count)
{
    const Plan& P = plan->p;
    if (n_calls < 0 || (n_calls > 0 && lens == nullptr) || zeros_fed == nullptr || count == nullptr) {
        set_err("simulate_flush: bad arguments");
        return -1;
    }
    for (const StageDesc& s : P.stages)
        if (s.kind == ST_FRAC_POLY && s.fasttiming) {
            set_err("simulate_flush: R8B_FASTTIMING plans cannot flush channels on their own");
            return -1;
        }
    if (target < 0 && P.trim_stage >= 0) {
        set_err(std::string("simulate_flush: ") + kTrimDefaultFlush);
        return -1;
    }
    Schedule sc;
    sc.init(&P);
    std::vector<StageCall> calls;
    long long n_in = 0, n_out = 0;
    for (int i = 0; i < n_calls; i++) {
        if (lens[i] < 0 || lens[i] > P.max_in_len) {
            set_err("simulate_flush: block length outside [0, MaxInLen]");
            return -1;
        }
        n_in += lens[i];
        n_out += sc.advance(lens[i], calls);
    }
    const long long T = target >= 0 ? target : flush_default_target(P, n_in);
    if (T < 0 || T - n_out > INT_MAX) {
        set_err("simulate_flush: target out of range");
        return -1;
    }
    if (P.passthrough) { // the input comes back as it is: the tail is T - E zeros
        *count = (int) std::max(0LL, T - n_out);
        *zeros_fed = *count;
        return 0;
    }
    FlushPlan f;
    plan_flush(sc, T, f, false); // counts only: no per-sub-step state is kept, whatever the target
    *zeros_fed = f.zeros;
    *count = f.count;
    return 0;
}

// ------------------------------------------------------------------------------------------

int r8bgpu_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

static r8bgpu_batch* create_front(const r8bgpu_plan* plan, int n_channels, int n_sh, int ndev)
{
    std::unique_ptr<r8bgpu_batch> b(new r8bgpu_batch);
    b->plan_copy = plan->p;
    b->plan = &b->plan_copy;
    b->n_ch = n_channels;
    b->device = -1;
    b->front.reset(new ShardFront);
    ShardFront& F = *b->front;
    const int per = (n_channels + n_sh - 1) / n_sh; // ceil(C / G) channels per shard, the last one takes the rest
    for (int s = 0; s * per < n_channels; s++) {
        const int c0 = s * per, n = std::min(per, n_channels - c0), dev = s % ndev;
        F.shards.emplace_back(r8bgpu_batch_create(plan, n, dev));
        if (F.shards.back() == nullptr) return nullptr; // (b's destructor releases the shards made so far)
        F.ch0.push_back(c0);
        F.device.push_back(dev);
        F.numa.push_back(gpu_numa_node(dev));
    }
    F.pool.reset(new ShardPool(F.numa));
    return b.release();
}

// A call on a multi-device batch: every shard runs its own channel range of the caller's buffers on its own worker
// thread, stream set and PCIe link.  plan(shard batch, shard index) first checks the call on every shard without
// changing anything, and every shard must accept it before run(shard batch, shard index) runs on any (shards that ran
// ragged calls may be in different states), so that a refused call changes nothing.  The shards return the same count.
// A failed run fails the call (the shards' schedules then disagree: the caller must clear()).
static int front_call(r8bgpu_batch* b, const std::function<bool(r8bgpu_batch*, int)>& plan,
                      const std::function<int(r8bgpu_batch*, int)>& run)
{
    ShardFront& F = *b->front;
    for (size_t s = 0; s < F.shards.size(); s++)
        if (!plan(F.shards[s].get(), (int) s)) return -1;
    std::vector<std::string> errs;
    const std::function<int(int)> job = [&](int s) { return run(F.shards[(size_t) s].get(), s); };
    const std::function<std::string()> err = [] { return g_err; };
    const std::vector<int> r = F.pool->run_all(job, &errs, err);
    for (size_t s = 0; s < r.size(); s++)
        if (r[s] < 0) {
            set_err("shard " + std::to_string(s) + " (device " + std::to_string(F.device[s]) + "): " + errs[s]);
            return -1;
        }
    for (size_t s = 1; s < r.size(); s++)
        if (r[s] != r[0]) {
            set_err("multi-device batch: shards disagree on the output count");
            return -1;
        }
    return r.empty() ? 0 : r[0];
}

r8bgpu_batch* r8bgpu_batch_create(const r8bgpu_plan* plan, int n_channels, int device)
{
    if (plan == nullptr || n_channels <= 0 || n_channels > 65535) {
        set_err("batch_create: need a plan and 1..65535 channels");
        return nullptr;
    }
    int ndev = 0;
    if (!cuda_ok(cudaGetDeviceCount(&ndev), "batch_create: cudaGetDeviceCount") || ndev == 0) {
        if (g_err.empty()) set_err("batch_create: no CUDA device (this engine has no CPU fallback)");
        return nullptr;
    }
    if (device == R8BGPU_DEVICE_ALL) {
        // shard over every visible device (R8BGPU_FORCE_SHARDS=n: n shards dealt round-robin to the devices -- lets a
        // one-GPU box exercise the multi-device path)
        int n_sh = ndev;
        if (const char* e = getenv("R8BGPU_FORCE_SHARDS")) n_sh = atoi(e) > 0 ? atoi(e) : ndev;
        if (n_sh > n_channels) n_sh = n_channels;
        if (n_sh > 1) return create_front(plan, n_channels, n_sh, ndev);
        device = 0;
        if (ndev > 1 && !cuda_ok(cudaGetDevice(&device), "batch_create: cudaGetDevice")) return nullptr;
    }
    if (device < 0 && !cuda_ok(cudaGetDevice(&device), "batch_create: cudaGetDevice")) return nullptr;
    if (device >= ndev) {
        set_err("batch_create: device index out of range");
        return nullptr;
    }
    DeviceGuard g(device);
    if (!g.ok) {
        set_err("batch_create: cudaSetDevice failed");
        return nullptr;
    }
    std::unique_ptr<r8bgpu_batch> b(new r8bgpu_batch);
    b->plan_copy = plan->p;
    b->plan = &b->plan_copy;
    b->n_ch = n_channels;
    b->device = device;
    b->sched.init(b->plan);
    b->pass_n.assign((size_t) n_channels, 0);
    if (b->plan->trim_stage >= 0) b->trim.assign((size_t) n_channels, 1.0);
    if (!cuda_ok(cudaDeviceGetAttribute(&b->n_sm, cudaDevAttrMultiProcessorCount, device), "batch_create: SM count")) return nullptr;
    const FusedKnobs knobs = fused_knobs_env();
    const HbKnobs hknobs = hb_knobs_env();
    b->f2_flags = knobs.f2_flags;
    b->f2_flags_env = knobs.f2_flags_env;
    const auto& st = b->plan->stages;
    b->dev.resize(st.size());
    std::vector<FusedPlan> fplan(st.size());
    for (size_t i = 0; i < st.size(); i++) fplan[i] = plan_fused_stage(st, i, knobs);
    for (size_t i = 0; i < st.size(); i++) {
        const StageDesc& s = st[i];
        StageDev& d = b->dev[i];
        const FusedPlan& fp = fplan[i];
        const long long emit_in = (i == 0) ? 0 : st[i - 1].max_out_len;
        if (fp.geom.ok) {
            d.f2_poly = fp.poly_v2;
            d.fused_with_next = true;
            b->dev[i + 1].fused_into_prev = true;
            d.fgeom = fp.geom;
            d.yl = fp.geom.yl;
            d.yr = fp.geom.yr;
            d.span_max = fp.geom.span_max;
            d.ysh = fp.geom.ysh;
        }
        long long extra_history = 0;
        if ((s.kind == ST_HBUP || s.kind == ST_HBDOWN) && !d.fused_into_prev) {
            const HbRunPlan hr = plan_hb_run(st, i, hknobs);
            const size_t c = (size_t) hr.n_stages;
            for (size_t k = 1; k < c; k++) b->dev[i + k].fused_into_prev = true;
            if (c >= 2 && s.kind == ST_HBUP) {
                d.casc_len = (int) c;
                d.up_casc = hr.up;
                d.up_casc_smem = hr.smem_bytes;
            } else if (c >= 2) {
                d.down_casc_len = (int) c;
                d.down_casc = hr.down;
                d.down_casc_smem = hr.smem_bytes;
                // the cascade recomputes intermediate samples of earlier calls from the source: keep its whole reach
                extra_history = 2LL * hr.down.back[0] + (2LL << c) + 64;
            }
        }
        if (d.fused_into_prev) {
            d.ring_cap = 0; // the link stream lives only in shared memory
        } else {
            d.ring_cap = next_pow2(std::max<long long>(s.src_history, extra_history) + emit_in + 64);
            if (!d.ring.alloc(b->dev_bytes, (size_t) d.ring_cap * (size_t) n_channels, "batch_create: cudaMalloc(ring)")) return nullptr;
        }
        if (s.kind == ST_BLOCKCONV) {
            const BcPlan bp = plan_blockconv_stage(s, fp, n_channels, bcl_scratch_cap_env());
            if (!bp.err.empty()) {
                set_err("batch_create: " + bp.err);
                return nullptr;
            }
            d.virt_up = bp.t.virt_up;
            d.lg = bp.t.lg;
            d.fft_log2 = bp.t.fft_log2;
            d.large = bp.t.large;
            if (fp.copy) {
                d.f2_copy = true;
                d.fgeom = FusedGeom();
                d.fgeom.ok = true;
                d.fgeom.up = 2;
                d.fgeom.lg = d.lg;
                d.fgeom.span_max = (2 * (4096 - 2 * d.lg)) & ~3;
            }
            std::vector<double2> spec, tw;
            if (d.large) {
                std::vector<double2> tw_m;
                build_spectrum_large(s, d.fft_log2, spec, tw, tw_m, &d.nyq_gain);
                if (!d.tw_m.upload(b->dev_bytes, tw_m, "cudaMalloc(tw_m)", "copy tw_m")) return nullptr;
                d.scratch_pairs = (long long) bp.group_ch * (bp.scratch_tiles / 2);
                const size_t sb = (size_t) bp.group_ch * (size_t) bp.scratch_per_ch;
                if (!d.scratch.alloc(b->dev_bytes, sb / sizeof(double2), "batch_create: cudaMalloc(large-tile scratch)")) return nullptr;
            } else {
                build_spectrum(s, d.fft_log2, spec, tw, &d.nyq_gain);
            }
            if (!d.spec.upload(b->dev_bytes, spec, "cudaMalloc(spec)", "copy spec") ||
                !d.tw.upload(b->dev_bytes, tw, "cudaMalloc(tw)", "copy tw"))
                return nullptr;
            if (d.fused_with_next || d.f2_copy) { // conflict-free [q][r] twiddle tables, one 8 KB bulk copy per CTA in the v2 kernel
                if (!d.tw_tab.upload(b->dev_bytes, build_tw_tab(tw), "cudaMalloc(tw_tab)", "copy tw_tab")) return nullptr;
                if (d.fgeom.up == 1 && !d.c_tab.upload(b->dev_bytes, build_c_tab(spec, tw, 1), "cudaMalloc(c_tab)", "copy c_tab"))
                    return nullptr;
                if (d.fgeom.up == 2) {
                    if (!d.cd_tab.upload(b->dev_bytes, build_cd_tab(spec, tw), "cudaMalloc(cd_tab)", "copy cd_tab")) return nullptr;
                    if (fp.cs && !d.cs_tab.upload(b->dev_bytes, build_cs_tab(s, tw), "cudaMalloc(cs_tab)", "copy cs_tab"))
                        return nullptr;
                }
                if (d.fused_with_next && d.fgeom.up == 2 &&
                    !d.c_tab_v1.upload(b->dev_bytes, build_c_tab_v1(spec), "cudaMalloc(c_tab_v1)", "copy c_tab_v1"))
                    return nullptr;
            }
        } else if (s.kind == ST_FRAC_WHOLE || s.kind == ST_FRAC_POLY) {
            const FracPlan fr = plan_frac_stage(*b->plan, i);
            if (!fr.err.empty()) {
                set_err("batch_create: " + fr.err);
                return nullptr;
            }
            d.frac_tile_fixed = fr.tile_fixed;
            d.frac_tile_ragged = fr.tile_ragged;
            if (!d.bank.upload(b->dev_bytes, s.bank.table, "cudaMalloc(bank)", "copy bank")) return nullptr;
            if (s.kind == ST_FRAC_POLY && s.fasttiming) {
                const size_t cap = (size_t) s.max_out_len + 16;
                if (!d.ft_dp.create(b->dev_bytes, cap, "cudaMalloc(ft)", "cudaMallocHost(ft)", "cudaEventCreate(ft)") ||
                    !d.ft_fpos.create(b->dev_bytes, cap, "cudaMalloc(ft)", "cudaMallocHost(ft)", "cudaEventCreate(ft)"))
                    return nullptr;
            }
            if (s.kind == ST_FRAC_WHOLE) {
                // per output phase r: floor(r*InStep/OutStep) and the bank row (r*InStep) % OutStep; grouped bank for
                // the fused kernels: IR consecutive phases share one y window
                // (the tensor-path interpolation of the v2 kernel works on groups of exactly 8 phases)
                const FusedPlan* pp = i > 0 && fplan[i - 1].whole ? &fplan[i - 1] : nullptr;
                GroupBank plain;
                if (pp == nullptr) plain = build_group_bank(s, choose_group_ir(s), false);
                const GroupBank& B = pp != nullptr ? (pp->tc_bank ? pp->tc : pp->fma) : plain;
                d.bank_frag_order = pp != nullptr && pp->tc_bank;
                if (!d.phase_off.upload(b->dev_bytes, B.off, "cudaMalloc(phase)", "copy phase") ||
                    !d.phase_row.upload(b->dev_bytes, B.row, "cudaMalloc(phase)", "copy phase") ||
                    !d.gbank.upload(b->dev_bytes, B.gb, "cudaMalloc(gbank)", "copy gbank") ||
                    !d.goff.upload(b->dev_bytes, B.go, "cudaMalloc(goff)", "copy goff"))
                    return nullptr;
                d.gbank_smem_len = B.n_groups * B.smaxp * B.ir;
                d.ir = B.ir;
                d.gbank_len = (int) B.gb.size();
                d.smaxp = B.smaxp;
                d.bank_in_smem = pp != nullptr && pp->bank_in_smem ? 1 : 0;
                if (pp != nullptr && (pp->kernel == R8BGPU_FUSED_F2_TC || pp->kernel == R8BGPU_FUSED_F2_FMA))
                    b->dev[i - 1].f2_ok = true;
            }
        }
    }
    r8bgpu_batch* raw = b.release();
    if (r8bgpu_batch_clear(raw) != 0) {
        delete raw;
        return nullptr;
    }
    return raw;
}

void r8bgpu_batch_destroy(r8bgpu_batch* batch) { delete batch; }
int r8bgpu_batch_channels(const r8bgpu_batch* b) { return b->n_ch; }

unsigned long long r8bgpu_batch_kernel_launches(const r8bgpu_batch* b)
{
    unsigned long long n = b->front ? 0 : b->launches; // a mixed batch: its conversions, plus its parts' chains
    if (const auto* subs = sub_batches(b))
        for (const auto& sb : *subs) n += sb->launches;
    return n;
}
unsigned long long r8bgpu_batch_device_bytes(const r8bgpu_batch* b)
{
    unsigned long long n = b->front ? 0 : b->dev_bytes; // a mixed batch: its records and host-form blocks, plus its parts
    if (const auto* subs = sub_batches(b))
        for (const auto& sb : *subs) n += sb->dev_bytes;
    return n;
}
int r8bgpu_batch_shard_count(const r8bgpu_batch* b) { return b->front ? (int) b->front->shards.size() : 1; }
int r8bgpu_batch_shard_info(const r8bgpu_batch* b, int shard, int* device, int* first_channel, int* n_channels, int* numa_node)
{
    if (shard < 0 || shard >= r8bgpu_batch_shard_count(b)) {
        set_err("batch_shard_info: shard index out of range");
        return -1;
    }
    if (!b->front) {
        if (device) *device = b->device;
        if (first_channel) *first_channel = 0;
        if (n_channels) *n_channels = b->n_ch;
        if (numa_node) *numa_node = gpu_numa_node(b->device);
        return 0;
    }
    const ShardFront& F = *b->front;
    if (device) *device = F.device[(size_t) shard];
    if (first_channel) *first_channel = F.ch0[(size_t) shard];
    if (n_channels) *n_channels = F.shards[(size_t) shard]->n_ch;
    if (numa_node) *numa_node = F.numa[(size_t) shard];
    return 0;
}
r8bgpu_batch* r8bgpu_batch_shard(r8bgpu_batch* b, int shard)
{
    if (shard < 0 || shard >= r8bgpu_batch_shard_count(b)) {
        set_err("batch_shard: shard index out of range");
        return nullptr;
    }
    return b->front ? b->front->shards[(size_t) shard].get() : b;
}

void* r8bgpu_batch_host_alloc(const r8bgpu_batch* b, size_t samples_per_channel, int sample_bytes)
{
    if (b == nullptr || sample_bytes <= 0 || samples_per_channel == 0) {
        set_err("batch_host_alloc: bad arguments");
        return nullptr;
    }
    const size_t row = samples_per_channel * (size_t) sample_bytes;
    std::vector<NumaRange> ranges;
    const int n_sh = r8bgpu_batch_shard_count(b);
    for (int s = 0; s < n_sh; s++) {
        int c0 = 0, n = 0, node = -1;
        r8bgpu_batch_shard_info(b, s, nullptr, &c0, &n, &node);
        ranges.push_back({(size_t) c0 * row, (size_t) n * row, node});
    }
    void* p = numa_host_alloc(row * (size_t) b->n_ch, ranges);
    if (p == nullptr) set_err("batch_host_alloc: mmap / cudaHostRegister failed");
    return p;
}

int r8bgpu_batch_set_timing(r8bgpu_batch* b, int enable)
{
    if (const auto* subs = sub_batches(b)) {
        int rc = 0;
        for (const auto& sb : *subs) rc |= r8bgpu_batch_set_timing(sb.get(), enable);
        return rc;
    }
    DeviceGuard g(b->device);
    b->events.clear();
    // (one more slot: the DSD modulator, K8, timed as the stage after the last)
    b->stage_ms.assign(b->plan->stages.size() + 1, 0.0);
    b->stage_launches.assign(b->plan->stages.size() + 1, 0);
    b->timing = enable != 0;
    return 0;
}

// Synchronises the stream, folds the pending event pairs into per-stage totals and returns the
// accumulated device time (ms) of `stage` since timing was enabled; *launches = kernel launches.
double r8bgpu_batch_stage_time_ms(r8bgpu_batch* b, int stage, unsigned long long* launches)
{
    if (b->front) { // the shards run side by side: report the slowest one
        double worst = 0.0;
        for (const auto& sb : b->front->shards) {
            const double t = r8bgpu_batch_stage_time_ms(sb.get(), stage, launches);
            if (t < 0.0) return t;
            if (t > worst) worst = t;
        }
        return worst;
    }
    if (b->mixed) {
        set_err("stage_time_ms: a stage index means nothing across the plans of a mixed batch; ask its parts "
                "(r8bgpu_batch_part())");
        return -1.0;
    }
    if (stage < 0 || stage >= (int) b->stage_ms.size()) {
        set_err("stage_time_ms: timing not enabled or bad stage");
        return -1.0;
    }
    DeviceGuard g(b->device);
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "stage_time_ms: sync")) return -1.0;
    for (auto& e : b->events) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, e.a, e.b) == cudaSuccess) {
            b->stage_ms[(size_t) e.stage] += ms;
            b->stage_launches[(size_t) e.stage]++;
        }
    }
    b->events.clear();
    if (launches) *launches = b->stage_launches[(size_t) stage];
    return b->stage_ms[(size_t) stage];
}

// Which kernel executes plan stage `stage`, and how many consecutive plan stages it covers
// (0 = this stage is folded into the kernel of an earlier stage).
int r8bgpu_batch_stage_kernel(const r8bgpu_batch* b, int stage, char* name, int cap)
{
    if (b->front) return r8bgpu_batch_stage_kernel(b->front->shards[0].get(), stage, name, cap);
    if (b->mixed) {
        set_err("stage_kernel: a stage index means nothing across the plans of a mixed batch; ask its parts "
                "(r8bgpu_batch_part())");
        return -1;
    }
    if (stage < 0 || stage >= (int) b->plan->stages.size()) {
        set_err("stage_kernel: bad stage index");
        return -1;
    }
    const StageDev& d = b->dev[(size_t) stage];
    const StageDesc& s = b->plan->stages[(size_t) stage];
    const char* nm = "";
    int span = 1;
    if (b->diverged) { // calls run ragged: every stage on its own kernel's per-channel-record instantiation
        switch (s.kind) {
        case ST_BLOCKCONV: nm = d.large ? "k_bcl_gather_ragged+k_bcl_conv+k_bcl_scatter_ragged" : "k_blockconv<ragged>"; break;
        case ST_FRAC_WHOLE: nm = "k_frac<false,ragged>"; break;
        case ST_FRAC_POLY: nm = "k_frac<true,ragged>"; break;
        case ST_HBUP: nm = "k_hbup<ragged>"; break;
        default: nm = "k_hbdown<ragged>"; break;
        }
    } else if (d.fused_into_prev) {
        nm = "(fused)";
        span = 0;
    } else if (d.fused_with_next) {
        nm = d.f2_ok ? "k_up2_frac2" : d.f2_poly ? "k_up2_frac2<poly>|k_up2_frac" : "k_up2_frac";
        span = 2;
    } else if (d.down_casc_len >= 2) {
        nm = "k_hbdown_cascade";
        span = d.down_casc_len;
    } else if (d.casc_len >= 2) {
        nm = "k_hbup_cascade";
        span = d.casc_len;
    } else {
        switch (s.kind) {
        case ST_BLOCKCONV: nm = d.f2_copy ? "k_up2_frac2<copy>" : d.large ? "k_bcl_gather+k_bcl_conv+k_bcl_scatter" : "k_blockconv"; break;
        case ST_FRAC_WHOLE: nm = "k_frac<false>"; break;
        case ST_FRAC_POLY: nm = "k_frac<true>"; break;
        case ST_HBUP: nm = "k_hbup"; break;
        default: nm = "k_hbdown"; break;
        }
    }
    if (name != nullptr && cap > 0) {
        strncpy(name, nm, (size_t) cap - 1);
        name[cap - 1] = 0;
    }
    return span;
}

int r8bgpu_batch_last_variant(const r8bgpu_batch* b, int stage, char* name, int cap)
{
    if (b->front) return r8bgpu_batch_last_variant(b->front->shards[0].get(), stage, name, cap);
    if (b->mixed) {
        set_err("last_variant: a stage index means nothing across the plans of a mixed batch; ask its parts "
                "(r8bgpu_batch_part())");
        return -1;
    }
    if (stage < 0 || stage >= (int) b->plan->stages.size()) {
        set_err("last_variant: bad stage index");
        return -1;
    }
    const StageDev& d = b->dev[(size_t) stage];
    const FusedVariant& v = d.last_variant;
    auto tf = [](int x) { return x ? "true" : "false"; };
    char buf[128] = "";
    if (d.casc_variant) {
        const bool up = d.casc_len >= 2;
        const int n = up ? d.up_casc.n_stages : d.down_casc.n_stages;
        const int* nt = up ? d.up_casc.ntaps : d.down_casc.ntaps;
        int o = snprintf(buf, sizeof buf, "%s stages=%d taps=", up ? "k_hbup_cascade" : d.casc_variant == 2 ? "k_hbdown_cascade<DSD>" : "k_hbdown_cascade", n);
        for (int k = 0; k < n; k++) o += snprintf(buf + o, sizeof buf - (size_t) o, k ? "/%d" : "%d", nt[k]);
        if (up) snprintf(buf + o, sizeof buf - (size_t) o, " last2=%d w=%d", d.up_casc.fuse_last2, d.up_casc.w);
        else snprintf(buf + o, sizeof buf - (size_t) o, " w=%d", d.down_casc.w);
    } else if (!d.unfused_variant.empty())
        snprintf(buf, sizeof buf, "%s", d.unfused_variant.c_str());
    else if (v.kernel == 2)
        snprintf(buf, sizeof buf, "k_up2_frac2<%d,%s,%d,%s,%d,%s,%s,%s,%s> mbu=%d", v.ir, tf(v.pad), v.glog, tf(v.tc), v.up,
                 tf(v.copy), tf(v.poly), tf(v.cs), tf(v.lin), v.mbu);
    else if (v.kernel == 1) {
        const int o = snprintf(buf, sizeof buf, "k_up2_frac<%d,%d,%s,%s>", v.mode, v.ir, tf(v.pad), tf(v.bank));
        if (v.mode == 1)
            snprintf(buf + o, sizeof buf - (size_t) o, " tiles=%d span=%d dir=%s rows=%d stride=%d chunks=%d N=%d", v.tiles,
                     v.span, v.dir > 0 ? "+1" : v.dir < 0 ? "-1" : "0", v.rows, v.stride, v.chunks, v.n);
    }
    if (name != nullptr && cap > 0) {
        strncpy(name, buf, (size_t) cap - 1);
        name[cap - 1] = 0;
    }
    return (int) strlen(buf);
}

int r8bgpu_batch_set_stream(r8bgpu_batch* b, void* stream)
{
    if (b->front) {
        if (stream == nullptr) return 0;
        set_err("batch_set_stream: a multi-device batch has one stream per shard (use r8bgpu_batch_shard())");
        return -1;
    }
    if ((cudaStream_t) stream != b->stream) {
        // work queued on the old stream (previous calls share the rings with the next ones) must be ordered before anything
        // the new stream runs: an event recorded there, waited for here
        DeviceGuard g(b->device);
        Event ev;
        if (cudaEventCreateWithFlags(ev.put(), cudaEventDisableTiming) == cudaSuccess) {
            cudaEventRecord(ev, b->stream);
            cudaStreamWaitEvent((cudaStream_t) stream, ev, 0);
        }
    }
    b->stream = (cudaStream_t) stream;
    return 0;
}

int r8bgpu_batch_clear(r8bgpu_batch* b)
{
    if (const auto* subs = sub_batches(b)) {
        int rc = 0;
        for (const auto& sb : *subs) rc |= r8bgpu_batch_clear(sb.get());
        if (b->mixed) {
            DeviceGuard g(b->device);
            if (!dither_clear_all(b, b->stream) || !dsd_clear(b, nullptr, 0, b->stream) ||
                !cuda_ok(cudaStreamSynchronize(b->stream), "batch_clear: sync"))
                rc = -1;
        }
        return rc == 0 ? 0 : -1;
    }
    DeviceGuard g(b->device);
    if (b->diverged && b->plan->trim_stage >= 0) {
        // channels with different trim factors stay apart: each restarts with its own factor
        std::vector<int> all((size_t) b->n_ch);
        for (int c = 0; c < b->n_ch; c++) all[(size_t) c] = c;
        b->rag.clear_channels(all.data(), b->n_ch);
        b->diverged = !b->rag.converged();
        if (!b->diverged) b->sched = b->rag.groups[0];
    } else {
        b->sched.clear();
        b->diverged = false;
    }
    std::fill(b->pass_n.begin(), b->pass_n.end(), 0LL);
    for (auto& d : b->dev) {
        if (d.ring == nullptr) continue;
        if (!cuda_ok(cudaMemsetAsync(d.ring, 0, (size_t) d.ring_cap * (size_t) b->n_ch * sizeof(double), b->stream),
                     "batch_clear: cudaMemsetAsync"))
            return -1;
    }
    if (!dither_clear_all(b, b->stream) || !dsd_clear(b, nullptr, 0, b->stream)) return -1;
    // clear() is rare; finishing it here keeps the device path (batch stream) and the host path
    // (internal pipeline streams) ordered without cross-stream events
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "batch_clear: sync")) return -1;
    return 0;
}

int r8bgpu_batch_sync(r8bgpu_batch* b)
{
    if (b->front) {
        int rc = 0;
        for (const auto& sb : b->front->shards) rc |= r8bgpu_batch_sync(sb.get());
        return rc == 0 ? 0 : -1;
    }
    DeviceGuard g(b->device);
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "batch_sync")) return -1;
    if (b->mixed)
        for (const auto& pb : b->mixed->parts)
            if (r8bgpu_batch_sync(pb.get()) != 0) return -1;
    return 0;
}

// With timing on, the events around stage `stage`'s launches on st: time_begin records the first, time_end the second
// and queues the pair for r8bgpu_batch_stage_time_ms.
static r8bgpu_batch::EvPair time_begin(r8bgpu_batch* b, int stage, cudaStream_t st)
{
    r8bgpu_batch::EvPair ev{stage, {}, {}};
    if (b->timing && cudaEventCreate(ev.a.put()) == cudaSuccess && cudaEventCreate(ev.b.put()) == cudaSuccess)
        cudaEventRecord(ev.a, st);
    else
        ev.a.reset();
    return ev;
}

static void time_end(r8bgpu_batch* b, r8bgpu_batch::EvPair& ev, cudaStream_t st)
{
    if (ev.a == nullptr) return;
    cudaEventRecord(ev.b, st);
    b->events.push_back(std::move(ev));
}

// R8B_FASTTIMING: ship this call's host-walked (position, fraction) sequence to the device, in stream order
// ahead of the kernels that read it.  Two pinned staging buffers alternate; an event guards their reuse.
static bool upload_fasttiming(r8bgpu_batch* b, cudaStream_t st)
{
    const Plan& P = *b->plan;
    for (size_t i = 0; i < P.stages.size(); i++) {
        const StageDesc& s = P.stages[i];
        if (s.kind != ST_FRAC_POLY || !s.fasttiming) continue;
        StageDev& d = b->dev[i];
        const StageCall& c = b->calls[i];
        const size_t n = c.ft_dp.size();
        if (n == 0) continue;
        int* dp = d.ft_dp.next("fasttiming upload");
        double* fpos = d.ft_fpos.next("fasttiming upload");
        if (dp == nullptr || fpos == nullptr) return false;
        memcpy(dp, c.ft_dp.data(), n * sizeof(int));
        memcpy(fpos, c.ft_fpos.data(), n * sizeof(double));
        if (!d.ft_dp.upload(0, n, st, "fasttiming upload") || !d.ft_fpos.upload(0, n, st, "fasttiming upload")) return false;
    }
    return true;
}

// Launches every kernel of one process() call (already scheduled in b->calls) for the channel range
// [ch0, ch0+nch) on stream st.  d_in / d_out point at the FIRST channel of that range.
// TypedIO: when the first / last kernel of the chain converts caller-side sample formats itself (fuses_input_format(),
// fuses_output_format()), d_in / d_out address planar samples of that format and the strides count samples.
struct TypedIO {
    int in_fmt = FMT_F64, out_fmt = FMT_F64;
    double in_scale = 1.0, out_scale = 1.0;
    const DitherCall* out_dither = nullptr; // flat TPDF in the stores (records of the call uploaded)
};

// The v2 fused kernel widens a planar typed block while it gathers its tiles / narrows in its tensor-path stores.
static bool fuses_input_format(const r8bgpu_batch* b)
{
    return !b->plan->passthrough && !b->dev.empty() && ((b->dev[0].fused_with_next && b->dev[0].f2_ok &&
           b->plan->stages[1].kind == ST_FRAC_WHOLE) || b->dev[0].f2_copy) && !getenv("R8BGPU_NO_FORMAT_FUSION");
}
static bool fuses_output_format(const r8bgpu_batch* b)
{
    const size_t ns = b->dev.size();
    return !b->plan->passthrough && ns >= 2 && b->plan->stages[ns - 1].kind == ST_FRAC_WHOLE && b->dev[ns - 1].fused_into_prev &&
           b->dev[ns - 2].f2_ok && b->dev[ns - 1].bank_frag_order && !getenv("R8BGPU_NO_FORMAT_FUSION");
}

// What r8bgpu_batch_last_variant names for the unfused kernels of a lock-step call: the instantiation and its call fields.
static std::string blockconv_variant(const BlockConvParams& p)
{
    char buf[128];
    snprintf(buf, sizeof buf, "k_blockconv M=%d up=%d src_up=%d down=%d trunc=%d tiles=%d", 1 << p.fft_log2, p.up, p.src_up,
             p.down, p.trunc, p.n_tiles);
    return buf;
}

static std::string bcl_variant(const BlockConvParams& p, int group_ch, int n_ch)
{
    char buf[128];
    snprintf(buf, sizeof buf, "k_bcl M=%d R0=%d src_up=%d down=%d trunc=%d tiles=%d groups=%d", 1 << p.fft_log2,
             1 << (p.fft_log2 - 12), p.src_up, p.down, p.trunc, p.n_tiles, (n_ch + group_ch - 1) / group_ch);
    return buf;
}

static std::string frac_variant(const StageDesc& s, int tile)
{
    char buf[96];
    snprintf(buf, sizeof buf, "k_frac poly=%d tile=%d flen=%d", s.kind == ST_FRAC_POLY ? 1 : 0, tile, s.bank.filter_len);
    return buf;
}

static void launch_call(r8bgpu_batch* b, const std::vector<StageCall>& calls, const double* d_in, size_t in_stride, int l, double* d_out,
                        size_t out_stride, int ch0, int nch, cudaStream_t st, const TypedIO& tio = TypedIO())
{
    const Plan& P = *b->plan;
    const size_t ns = P.stages.size();
    b->links_fresh = false;
    for (size_t i = 0; i < ns; i++) {
        const StageDesc& s = P.stages[i];
        const StageCall& c = calls[i];
        const StageDev& d = b->dev[i];
        if (d.fused_into_prev) continue; // handled together with the previous stage
        const bool fused = d.fused_with_next;
        const size_t last = fused ? i + 1 : (d.casc_len >= 2 ? i + (size_t) d.casc_len - 1 : d.down_casc_len >= 2 ? i + (size_t) d.down_casc_len - 1 : i); // stage whose output this launch produces
        if (calls[last].e1 <= calls[last].e0) continue;
        SrcView src;
        src.ring = d.ring + (long long) ch0 * d.ring_cap;
        src.ring_stride = d.ring_cap;
        src.ring_mask = d.ring_cap - 1;
        if (i == 0) {
            src.cur = d_in;
            src.cur_stride = (long long) in_stride;
            src.cur_base = c.n0;
            src.cur_fmt = tio.in_fmt;
            src.cur_scale = tio.in_scale;
        } else {
            src.cur = nullptr;
            src.cur_stride = 0;
            src.cur_base = LLONG_MAX;
        }
        src.avail = c.n1;
        DstView dst;
        if (last + 1 == ns) {
            dst.ptr = d_out;
            dst.stride = (long long) out_stride;
            dst.mask = -1;
            dst.base = calls[last].e0;
            dst.fmt = tio.out_fmt;
            dst.scale = tio.out_scale;
            dst.dither = tio.out_dither;
            dst.dither_ch0 = ch0;
        } else {
            dst.ptr = b->dev[last + 1].ring + (long long) ch0 * b->dev[last + 1].ring_cap;
            dst.stride = b->dev[last + 1].ring_cap;
            dst.mask = b->dev[last + 1].ring_cap - 1;
            dst.base = 0;
        }
        r8bgpu_batch::EvPair ev = time_begin(b, (int) i, st);
        if (d.down_casc_len >= 2) {
            HbDownCascParams p = d.down_casc;
            p.e0 = calls[last].e0;
            p.e1 = calls[last].e1;
            p.n_tiles = (int) ((p.e1 - p.e0 + p.w - 1) / p.w);
            launch_hbdown_cascade(p, d.down_casc_smem, src, dst, nch, st);
            b->dev[i].casc_variant = is_dsd_format(src.cur_fmt) ? 2 : 1;
            b->launches++;
        } else if (d.casc_len >= 2) {
            const int cl = d.casc_len;
            HbCascadeParams p = d.up_casc;
            p.e0 = calls[last].e0;
            p.e1 = calls[last].e1;
            p.a0 = p.e0 >> cl;
            const long long span = p.e1 - (p.a0 << cl);
            p.n_tiles = (int) ((span + ((long long) p.w << cl) - 1) / ((long long) p.w << cl));
            launch_hbup_cascade(p, d.up_casc_smem, src, dst, nch, st);
            b->dev[i].casc_variant = 1;
            b->launches++;
        } else if (fused) {
            const StageDesc& f = P.stages[i + 1];
            const StageCall& fc = calls[i + 1];
            const StageDev& fd = b->dev[i + 1];
            FusedParams p;
            memset(&p, 0, sizeof p);
            if (f.kind == ST_FRAC_WHOLE) {
                fused_whole_fields(p, f, fc.e0, fc.e1);
            } else {
                p.mode = 1;
                p.flen = f.bank.filter_len;
                p.fll = p.flen / 2 - 1;
                p.e0 = fc.e0;
                p.e1 = fc.e1;
                p.p_lo = fc.p0 & ~1LL; // even (positions are >= 0)
                p.p_hi = fc.p_last + 1;
                p.in_step = f.in_step;
                p.out_step = f.out_step;
            }
            // order-2 bank: the call's kernel, tiles and staged bank rows (plan_poly_call, r8b_hosttab.cpp)
            PolyCall pc;
            if (p.mode == 1)
                pc = plan_poly_call(f, d.fgeom, d.f2_poly, fc.ssr, fc.dsr, p.p_lo, p.p_hi, i == 0 ? (int) (c.n0 & 1) : -1,
                                    poly_knobs_env());
            const bool v2_poly = p.mode == 1 && pc.v2;
            const bool v2 = (d.f2_ok && p.mode == 0) || v2_poly;
            if (p.mode == 1) {
                p.n_tiles = pc.n_tiles;
                p.span = pc.span;
                p.p_lo = pc.p_lo;
            } else if (v2) {
                fused2_tiles(p, d.fgeom, i == 0 ? (int) (c.n0 & 1) : -1);
            } else {
                const long long range = p.p_hi - p.p_lo;
                long long nt = (range + d.span_max - 1) / d.span_max;
                if (nt > 1 && (nt & 1)) nt++;
                p.n_tiles = (int) nt;
                p.span = (int) (((range + nt - 1) / nt + 1) & ~1LL);
            }
            p.yl = d.yl;
            p.lg = d.lg;
            p.ysh = d.ysh;
            p.spec = d.spec;
            p.tw = d.tw;
            p.bank = fd.bank;
            p.bank_len = (int) f.bank.table.size();
            p.bank_in_smem = fd.bank_in_smem;
            p.gbank = fd.gbank;
            p.gbank_len = fd.gbank_len;
            p.smaxp = fd.smaxp;
            p.goff = fd.goff;
            p.ir = fd.ir;
            p.gbank_smem_len = fd.gbank_smem_len;
            {
                // store staging area behind the bank, if shared memory allows (whole stepping, 8-phase groups)
                const int used = fused_fixed_doubles() + (p.bank_in_smem ? ((p.gbank_smem_len + 1) & ~1) : 0);
                p.stage_off = (p.mode == 0 && p.ir == 8 && !getenv("R8BGPU_NO_STAGE") &&
                               (used + fused_stage_doubles()) * 8 <= 224 * 1024) ? used : 0;
            }
            p.phase_off = fd.phase_off;
            p.phase_row = fd.phase_row;
            p.fracs = f.bank.fracs;
            p.ssr = f.kind == ST_FRAC_POLY ? fc.ssr : f.src_rate; // order-2: this call's rates (a trimmed dsr)
            p.dsr = f.kind == ST_FRAC_POLY ? fc.dsr : f.dst_rate;
            p.in_counter0 = fc.in_counter0;
            p.in_pos_int0 = fc.in_pos_int0;
            p.in_pos_shift = fc.in_pos_shift;
            p.fpos0 = fc.fpos0;
            p.p0 = fc.p0;
            p.pos_dp = fd.ft_dp.d;
            p.pos_fpos = fd.ft_fpos.d;
            p.bank = fd.bank;
            if (p.mode == 1) {
                p.poly_dir = pc.poly_dir;
                p.poly_rows_cap = pc.poly_rows_cap;
                p.poly_row_stride = pc.poly_row_stride;
                p.poly_chunks = pc.poly_chunks;
                p.poly_n = pc.poly_n;
                p.ysh = pc.ysh;
            }
            if (p.poly_chunks < 1) p.poly_chunks = 1;
            if (b->prof == nullptr && getenv("R8BGPU_PROFILE") && b->prof.alloc(b->dev_bytes, 10, "profile: cudaMalloc"))
                cudaMemset(b->prof, 0, 10 * sizeof(unsigned long long));
            p.prof = b->prof;
#ifdef R8BGPU_EXPERIMENTS
            if (const char* e = getenv("R8BGPU_DEBUG")) p.debug = atoi(e);
#endif
            if (b->prof) {
                b->prof_ctas += (unsigned long long) (v2 ? p.n_tiles : (p.n_tiles + 1) / 2) * nch;
                b->prof_v2 = v2;
            }
            if (v2) {
                p.n_ch = nch;
                p.flags = b->f2_flags;
                p.tw_tab = d.tw_tab;
                p.c_tab = d.c_tab;
                p.cd_tab = d.cd_tab;
                p.cs_tab = d.cs_tab;
                p.up = d.fgeom.up;
                p.ylen = d.fgeom.up * 4096;
                if (!fd.bank_frag_order) p.flags &= ~4; // (the bank layout decides: see batch_create)
                // The two halves take turns at the tensor-path interpolation where phase C reads the filter spectrum from
                // shared memory: the transforms are then short enough that one half's run under the other's interpolation,
                // and the token keeps the halves out of phase (measured on H100, DESIGN section 8: 44100->96000 3-7 % faster;
                // 48000->44100 and the 1x pairs, which read the spectrum from L2, 1-2 % slower).  R8BGPU_F2_FLAGS decides alone.
                if (!b->f2_flags_env && !v2_poly && p.up != 1 && p.cs_tab != nullptr && (p.flags & 4)) p.flags |= 1;
                // (the staging area gives way to the spectrum table where both do not fit: staging changes no result bit)
                const bool cs = p.cs_tab != nullptr;
                p.stage_off = (p.ir == 8 && !(p.flags & 4) && fused2_smem_bytes(p.gbank_smem_len, cs, true) <= kFused2SmemMax &&
                               !getenv("R8BGPU_NO_STAGE")) ? fused2_stage_off(p.gbank_smem_len, cs) : 0;
                if (v2_poly) { // plain y layout; no grouped bank, no staging area in shared memory
                    p.ysh = 31;
                    p.gbank_smem_len = 0;
                    p.stage_off = 0;
                }
                p.glog = v2_poly ? 0 : fused2_choose_glog(p.span, f.in_step, f.out_step, p.ir);
                p.mbu = v2_poly ? 0 : fused2_choose_mbu(p.span, f.in_step, f.out_step);
                launch_up2_frac2(p, src, dst, b->n_sm, st, &b->dev[i].last_variant);
            } else {
                p.c_tab = d.c_tab_v1;
                launch_up2_frac(p, src, dst, nch, st, &b->dev[i].last_variant);
                if (p.mode == 1 && p.n_tiles > 0 && nch > 0) { // the call's order-2 fields, for r8bgpu_batch_last_variant
                    FusedVariant& v = b->dev[i].last_variant;
                    v.tiles = p.n_tiles;
                    v.span = p.span;
                    v.dir = p.poly_dir;
                    v.rows = p.poly_rows_cap;
                    v.stride = p.poly_row_stride;
                    v.chunks = p.poly_chunks;
                    v.n = p.poly_n;
                }
            }
            b->launches++;
        } else
        switch (s.kind) {
        case ST_BLOCKCONV: {
            if (d.f2_copy) {
                FusedParams fp;
                memset(&fp, 0, sizeof fp);
                fp.mode = 2;
                fp.e0 = c.e0;
                fp.e1 = c.e1;
                fp.p_lo = c.e0 & ~1LL;
                fp.p_hi = c.e1;
                fused2_tiles(fp, d.fgeom, i == 0 ? (int) (c.n0 & 1) : -1);
                fp.lg = d.lg;
                fp.ysh = 31;
                fp.spec = d.spec;
                fp.tw = d.tw;
                fp.tw_tab = d.tw_tab;
                fp.c_tab = d.c_tab;
                fp.cd_tab = d.cd_tab;
                fp.cs_tab = d.cs_tab;
                fp.up = 2;
                fp.ylen = 8192;
                fp.ir = 8;
                fp.out_step = 8; // one (unused) phase group
                fp.smaxp = 4;
                fp.n_ch = nch;
                fp.flags = b->f2_flags & 2;
                launch_up2_frac2(fp, src, dst, b->n_sm, st, &b->dev[i].last_variant);
                b->launches++;
                break;
            }
            BlockConvParams p;
            blockconv_call_fields(p, s, d.virt_up, d.lg, d.fft_log2, c.e0, c.e1);
            p.nyq_gain = d.nyq_gain;
            p.spec = d.spec;
            p.tw = d.tw;
            if (d.large) {
                BcLargeParams lp;
                lp.bc = p;
                lp.tw_m = d.tw_m;
                lp.scratch = d.scratch;
                // as many channels per launch group as the scratch holds this call's tile pairs (the sizing at batch_create
                // guarantees at least one)
                const long long pairs = (p.n_tiles + 1) / 2;
                lp.group_ch = (int) std::max(1LL, std::min((long long) nch, d.scratch_pairs / std::max(1LL, pairs)));
                b->launches += (unsigned long long) launch_blockconv_large(lp, src, dst, nch, st);
                if (p.n_tiles > 0 && nch > 0)
                    b->dev[i].unfused_variant = bcl_variant(p, lp.group_ch, nch);
                break;
            }
            launch_blockconv(p, src, dst, nch, st);
            if (p.n_tiles > 0 && nch > 0) b->dev[i].unfused_variant = blockconv_variant(p);
            b->launches++;
            break;
        }
        case ST_FRAC_WHOLE:
        case ST_FRAC_POLY: {
            FracParams p;
            memset(&p, 0, sizeof p);
            p.flen = s.bank.filter_len;
            p.fll = s.bank.filter_len / 2 - 1;
            p.e0 = c.e0;
            p.e1 = c.e1;
            p.bank = d.bank;
            p.in_step = s.in_step;
            p.out_step = s.out_step;
            p.fracs = s.bank.fracs;
            p.ssr = s.kind == ST_FRAC_POLY ? c.ssr : s.src_rate;
            p.dsr = s.kind == ST_FRAC_POLY ? c.dsr : s.dst_rate;
            p.in_counter0 = c.in_counter0;
            p.in_pos_int0 = c.in_pos_int0;
            p.in_pos_shift = c.in_pos_shift;
            p.fpos0 = c.fpos0;
            p.p0 = c.p0;
            p.pos_dp = d.ft_dp.d;
            p.pos_fpos = d.ft_fpos.d;
            const int tile = d.frac_tile_fixed > 0 ? d.frac_tile_fixed : frac_tile(p.ssr / p.dsr, p.flen);
            if (s.kind == ST_FRAC_WHOLE) launch_frac_whole(p, tile, src, dst, nch, st);
            else launch_frac_poly(p, tile, src, dst, nch, st);
            if (p.e1 > p.e0 && nch > 0) b->dev[i].unfused_variant = frac_variant(s, tile);
            b->launches++;
            break;
        }
        case ST_HBUP:
        case ST_HBDOWN: {
            HbParams p;
            memset(&p, 0, sizeof p);
            p.ntaps = s.hb_taps;
            p.e0 = c.e0;
            p.e1 = c.e1;
            for (int k = 0; k < s.hb_taps; k++) p.taps[k] = s.hb[(size_t) k];
            if (s.kind == ST_HBUP) launch_hbup(p, src, dst, nch, st);
            else launch_hbdown(p, src, dst, nch, st);
            b->launches++;
            break;
        }
        }
        time_end(b, ev, st);
    }
    // Keep the most recent input samples for the next calls.
    if (l > 0) {
        const StageCall& c0 = calls[0];
        const StageDev& d0 = b->dev[0];
        long long from = c0.n1 - d0.ring_cap;
        if (from < c0.n0) from = c0.n0;
        launch_save_tail(d_in, (long long) in_stride, c0.n0, from, c0.n1, d0.ring + (long long) ch0 * d0.ring_cap, d0.ring_cap,
                         d0.ring_cap - 1, nch, st, tio.in_fmt, tio.in_scale);
        b->launches++;
    }
}

// ---- channels with schedules of their own (ragged calls, per-channel clear) ------------------
// The schedule of each group of channels in the same state is advanced once per distinct block length; every stage then
// runs for all channels in one launch of its kernel's ragged instantiation, which reads each channel's call fields from
// a per-channel record (launch_ragged).

static bool has_fasttiming(const Plan& P)
{
    for (const StageDesc& s : P.stages)
        if (s.kind == ST_FRAC_POLY && s.fasttiming) return true;
    return false;
}

// The channels' schedules as they stand (a lock-step batch: every channel in b->sched).
static const RaggedSchedule& channel_schedules(r8bgpu_batch* b)
{
    if (!b->diverged) b->rag.init(b->sched, b->n_ch);
    return b->rag;
}

// Passthrough plans keep no schedule totals: their per-channel input totals (what a flush needs) are counted here for
// lock-step calls, and in adopt_step for ragged ones.
static void count_passthrough(r8bgpu_batch* b, int l)
{
    if (!b->plan->passthrough) return;
    for (long long& n : b->pass_n) n += l;
}

static void adopt_step(r8bgpu_batch* b, const RaggedSchedule::Step& step)
{
    if (b->plan->passthrough)
        for (int c = 0; c < b->n_ch; c++) b->pass_n[(size_t) c] += step.len[(size_t) step.key_of[(size_t) c]];
    b->rag.commit(step);
    b->diverged = !b->rag.converged();
    if (!b->diverged) b->sched = b->rag.groups[0];
}

// Validates a ragged call and plans it.  lockstep: a plain process() on a batch whose channels diverged -- every channel
// must produce the same count.
static bool plan_ragged(r8bgpu_batch* b, const char* what, const int* lens, bool have_in, bool have_out, int out_cap,
                        bool lockstep, RaggedSchedule::Step& step)
{
    const Plan& P = *b->plan;
    if (lens == nullptr) {
        set_err(std::string(what) + ": null lens");
        return false;
    }
    for (int c = 0; c < b->n_ch; c++) {
        if (lens[c] < 0 || lens[c] > P.max_in_len) {
            set_err(std::string(what) + ": lens[" + std::to_string(c) + "] outside [0, MaxInLen]");
            return false;
        }
        if (lens[c] > 0 && !have_in) {
            set_err(std::string(what) + ": null input");
            return false;
        }
    }
    if (has_fasttiming(P)) {
        set_err(std::string(what) + ": R8B_FASTTIMING plans upload one position table per call and run lock-step only");
        return false;
    }
    channel_schedules(b).plan_call(lens, step);
    for (size_t k = 0; k < step.count.size(); k++) {
        if (step.count[k] > out_cap || (step.count[k] > 0 && !have_out)) {
            set_err(std::string(what) + ": output capacity too small for this call");
            return false;
        }
        if (lockstep && step.count[k] != step.count[0]) {
            set_err(std::string(what) + ": this batch's channels have diverged (ragged calls or clear_channels) and would "
                    "produce " + std::to_string(step.count[0]) + " and " + std::to_string(step.count[k]) +
                    " samples; use r8bgpu_batch_process_ragged / _host_ragged, or clear the batch");
            return false;
        }
    }
    return true;
}

// ---- ragged launch sequence: every stage on its own kernel's RAG instantiation, all channels in one launch ----------

// Samples of stream j (the input of stage j) a ragged call may re-read below what has arrived, including what refilling
// the next fused-away link needs (link_need, below).
static long long link_need(const r8bgpu_batch* b, size_t j)
{
    const auto& st = b->plan->stages;
    long long need = st[j].src_history + 64;
    if (j + 1 < st.size() && b->dev[j + 1].fused_into_prev) {
        const StageDesc& s = st[j];
        const long long n = link_need(b, j + 1);
        if (s.kind == ST_BLOCKCONV) need += n * s.down / std::max(1, s.up) + 2LL * s.lp.kernel_len + 2;
        else if (s.kind == ST_HBUP) need += n / 2 + s.hb_taps + 2;
        else need += 2 * n + 2LL * s.hb_taps + 2;
    }
    return need;
}

// The links that lock-step calls keep in shared memory (fused pairs, half-band cascades) get rings of their own the first
// time a batch goes ragged; the per-channel records live next to them.
static bool ensure_ragged_state(r8bgpu_batch* b)
{
    const auto& st = b->plan->stages;
    const size_t ns = st.size();
    for (size_t j = 1; j < ns; j++) {
        StageDev& d = b->dev[j];
        if (d.ring != nullptr) continue;
        d.ring_cap = next_pow2(link_need(b, j) + st[j - 1].max_out_len + 64);
        const size_t n = (size_t) d.ring_cap * (size_t) b->n_ch;
        if (!d.ring.alloc(b->dev_bytes, n, "ragged: cudaMalloc(link ring)")) return false;
        if (!cuda_ok(cudaMemset(d.ring, 0, n * sizeof(double)), "ragged: cudaMemset(link ring)")) return false;
        b->links_fresh = false;
    }
    return b->rec.d != nullptr || b->rec.create(b->dev_bytes, (2 * ns + 1) * (size_t) b->n_ch, "ragged: cudaMalloc(records)",
                                                "ragged: cudaMallocHost(records)", "ragged: event");
}

// Records of stage i for every channel (cs[c]: channel c's StageCall); returns the uniform parameters of the largest
// channel in *bp (BlockConv) and its output count.
static long long fill_stage_records(const r8bgpu_batch* b, size_t i, const std::vector<const StageCall*>& cs, RaggedRec* h,
                                    BlockConvParams* bp)
{
    const StageDesc& s = b->plan->stages[i];
    const StageDev& dv = b->dev[i];
    const bool last = i + 1 == b->plan->stages.size();
    long long max_cnt = 0;
    int max_tiles = 0;
    memset(bp, 0, sizeof *bp);
    for (size_t c = 0; c < cs.size(); c++) {
        const StageCall& k = *cs[c];
        RaggedRec& r = h[c];
        memset(&r, 0, sizeof r);
        r.e0 = k.e0;
        r.e1 = k.e1;
        r.cur_base = i == 0 ? k.n0 : LLONG_MAX;
        r.avail = k.n1;
        r.dst_base = last ? k.e0 : 0;
        r.p0 = k.p0;
        r.in_pos_shift = k.in_pos_shift;
        r.fpos0 = k.fpos0;
        r.in_counter0 = k.in_counter0;
        r.in_pos_int0 = k.in_pos_int0;
        r.ssr = k.ssr;
        r.dsr = k.dsr;
        if (s.kind == ST_BLOCKCONV && k.e1 > k.e0) {
            BlockConvParams q;
            blockconv_call_fields(q, s, dv.virt_up, dv.lg, dv.fft_log2, k.e0, k.e1);
            r.m0 = q.m0;
            r.m1 = q.m1;
            r.n_tiles = q.n_tiles;
            r.adv = q.adv;
            if (q.n_tiles > max_tiles) {
                max_tiles = q.n_tiles;
                *bp = q;
            }
        }
        max_cnt = std::max(max_cnt, k.e1 - k.e0);
    }
    return max_cnt;
}

// One stage for every channel in one launch (the large-tile path: one per scratch group); d = the stage's device records.
static void launch_stage_ragged(r8bgpu_batch* b, size_t i, long long max_cnt, BlockConvParams bp, const RaggedRec* d,
                                const double* d_in, size_t in_stride, double* d_out, size_t out_stride, cudaStream_t st)
{
    const Plan& P = *b->plan;
    const StageDesc& s = P.stages[i];
    const StageDev& dv = b->dev[i];
    const int n_ch = b->n_ch;
    const bool last = i + 1 == P.stages.size();
    if (max_cnt <= 0) return;
    SrcView src;
    src.ring = dv.ring;
    src.ring_stride = dv.ring_cap;
    src.ring_mask = dv.ring_cap - 1;
    src.cur = i == 0 ? d_in : nullptr;
    src.cur_stride = i == 0 ? (long long) in_stride : 0;
    src.cur_base = LLONG_MAX;
    src.avail = 0;
    DstView dst;
    dst.ptr = last ? d_out : b->dev[i + 1].ring;
    dst.stride = last ? (long long) out_stride : b->dev[i + 1].ring_cap;
    dst.mask = last ? -1 : b->dev[i + 1].ring_cap - 1;
    dst.base = 0;
    r8bgpu_batch::EvPair ev = time_begin(b, (int) i, st);
    switch (s.kind) {
    case ST_BLOCKCONV: {
        bp.nyq_gain = dv.nyq_gain;
        bp.spec = dv.spec;
        bp.tw = dv.tw;
        if (dv.large) {
            BcLargeParams lp;
            lp.bc = bp;
            lp.tw_m = dv.tw_m;
            lp.scratch = dv.scratch;
            const long long pairs = (bp.n_tiles + 1) / 2;
            lp.group_ch = (int) std::max(1LL, std::min((long long) n_ch, dv.scratch_pairs / std::max(1LL, pairs)));
            b->launches += (unsigned long long) launch_blockconv_large(lp, src, dst, n_ch, st, d);
        } else {
            launch_blockconv(bp, src, dst, n_ch, st, d);
            b->launches++;
        }
        break;
    }
    case ST_FRAC_WHOLE:
    case ST_FRAC_POLY: {
        FracParams p;
        memset(&p, 0, sizeof p);
        p.flen = s.bank.filter_len;
        p.fll = s.bank.filter_len / 2 - 1;
        p.e0 = 0;
        p.e1 = max_cnt;
        p.bank = dv.bank;
        p.in_step = s.in_step;
        p.out_step = s.out_step;
        p.fracs = s.bank.fracs;
        // the kernel reads each channel's rates from its record; these size the tiles (input per output), so on a trim
        // plan they take the smallest factor's dsr, the most input per output any channel can read
        p.ssr = s.src_rate;
        p.dsr = (int) i == P.trim_stage ? P.trim_dsr(1.0 - P.max_trim) : s.dst_rate;
        if (s.kind == ST_FRAC_WHOLE) launch_frac_whole(p, dv.frac_tile_ragged, src, dst, n_ch, st, d);
        else launch_frac_poly(p, dv.frac_tile_ragged, src, dst, n_ch, st, d);
        b->launches++;
        break;
    }
    default: {
        HbParams p;
        memset(&p, 0, sizeof p);
        p.ntaps = s.hb_taps;
        p.e0 = 0;
        p.e1 = max_cnt;
        for (int k = 0; k < s.hb_taps; k++) p.taps[k] = s.hb[(size_t) k];
        if (s.kind == ST_HBUP) launch_hbup(p, src, dst, n_ch, st, d);
        else launch_hbdown(p, src, dst, n_ch, st, d);
        b->launches++;
        break;
    }
    }
    time_end(b, ev, st);
}

// The refill of the links that lock-step calls keep in shared memory (refill_launch): their stages' records in slots
// [0, ns) of h, from the channels' schedules `before`, and each stage's largest count and uniform parameters.
static void fill_refill_records(const r8bgpu_batch* b, const RaggedSchedule& before, RaggedRec* h, long long* cnt,
                                BlockConvParams* bp)
{
    const size_t ns = b->plan->stages.size();
    const size_t n_ch = (size_t) b->n_ch;
    std::vector<std::vector<StageCall>> rc(before.groups.size());
    for (size_t g = 0; g < before.groups.size(); g++) {
        const Schedule& S = before.groups[g];
        rc[g].assign(ns, StageCall());
        for (size_t j = 0; j + 1 < ns; j++) {
            StageCall& c = rc[g][j];
            c.n0 = c.n1 = S.n_in[j];
            c.e0 = c.e1 = S.n_out[j];
            if (b->dev[j + 1].fused_into_prev) c.e0 = std::max(0LL, c.e1 - link_need(b, j + 1));
        }
    }
    std::vector<const StageCall*> cs(n_ch);
    for (size_t j = 0; j + 1 < ns; j++) {
        if (!b->dev[j + 1].fused_into_prev) continue;
        for (size_t c = 0; c < n_ch; c++) cs[c] = &rc[(size_t) before.group_of[c]][j];
        cnt[j] = fill_stage_records(b, j, cs, h + j * n_ch, &bp[j]);
    }
}

static void refill_launch(r8bgpu_batch* b, const long long* cnt, const BlockConvParams* bp, cudaStream_t st)
{
    const size_t ns = b->plan->stages.size();
    for (size_t j = 0; j + 1 < ns; j++)
        if (b->dev[j + 1].fused_into_prev)
            launch_stage_ragged(b, j, cnt[j], bp[j], b->rec.d + j * (size_t) b->n_ch, nullptr, 0, nullptr, 0, st);
    b->links_fresh = true;
}

// Typed buffers around a ragged chain (r8bgpu_batch_process_ragged_fmt): one conversion pass in front of the first stage
// and one behind the last, each channel over its own extent, taken from the call's records.
struct RaggedConv {
    const r8bgpu_buffer* in = nullptr;  // widened into the chain's input block d_in first (nullptr: d_in is the caller's)
    const r8bgpu_buffer* out = nullptr; // narrowed from the chain's output block d_out last (nullptr: d_out is the caller's)
    int max_len = 0, max_count = 0;     // the largest block length and count of the call
};

// One sub-step of a flush (r8bgpu_batch_flush) through the ragged chain.  Channel c's first stage reads its history
// ring below zero_from[c] (its real input total) and silence from there on: the record's `avail` is set to it and the
// record has no input block, so no zero block exists anywhere.  Its last stage writes output e at (e - out_base[c]) of
// the channel's row, so the sub-steps' pieces land one after another.  No channel keeps history: the flushed channels
// are cleared afterwards and the others take no input.
struct FlushView {
    const std::vector<long long>* zero_from;
    const std::vector<long long>* out_base;
};

// The whole chain of one ragged call (planned in `step`; `before` = the channels' schedules before it) for every channel
// in one launch per stage; d_in / d_out address channel 0.  When lock-step calls ran since the last ragged call, the
// links they keep in shared memory are first recomputed into their rings from the stage in front of them: the newest
// link_need() samples of each channel's link stream, read from history only.  cv (optional): conversions of typed
// buffers into d_in and out of d_out, which are then the batch's staging blocks.
static bool launch_ragged(r8bgpu_batch* b, const RaggedSchedule& before, const RaggedSchedule::Step& step, const double* d_in,
                          size_t in_stride, double* d_out, size_t out_stride, cudaStream_t st, const RaggedConv* cv = nullptr,
                          const FlushView* fv = nullptr)
{
    if (!ensure_ragged_state(b)) return false;
    const size_t ns = b->plan->stages.size();
    const size_t n_ch = (size_t) b->n_ch;
    RaggedRec* h = b->rec.next("ragged: records"); // its last upload is done
    if (h == nullptr) return false;
    std::vector<const StageCall*> cs(n_ch);
    std::vector<long long> cnt(2 * ns, 0);
    std::vector<BlockConvParams> bp(2 * ns);
    const bool refill = !b->links_fresh;
    if (refill) fill_refill_records(b, before, h, cnt.data(), bp.data()); // (refill and call records go up in one copy)
    for (size_t i = 0; i < ns; i++) {
        for (size_t c = 0; c < n_ch; c++) cs[c] = &step.calls[(size_t) step.key_of[c]][i];
        cnt[ns + i] = fill_stage_records(b, i, cs, h + (ns + i) * n_ch, &bp[ns + i]);
    }
    if (fv != nullptr)
        for (size_t c = 0; c < n_ch; c++) {
            RaggedRec& first = h[ns * n_ch + c];
            first.cur_base = LLONG_MAX;
            first.avail = std::min(first.avail, (*fv->zero_from)[c]);
            h[(2 * ns - 1) * n_ch + c].dst_base = (*fv->out_base)[c];
        }
    // history copy: each channel keeps the newest samples of its own block
    long long tail = 0;
    RaggedRec* ht = h + 2 * ns * n_ch;
    for (size_t c = 0; c < n_ch; c++) {
        const StageCall& c0 = step.calls[(size_t) step.key_of[c]][0];
        memset(&ht[c], 0, sizeof ht[c]);
        ht[c].m1 = c0.n1;
        ht[c].m0 = fv != nullptr ? c0.n1 : std::max(c0.n0, c0.n1 - b->dev[0].ring_cap);
        ht[c].cur_base = c0.n0;
        tail = std::max(tail, ht[c].m1 - ht[c].m0);
    }
    if (!b->rec.upload(0, (2 * ns + 1) * n_ch, st, "ragged: record upload")) return false;
    if (cv != nullptr && cv->in != nullptr && cv->max_len > 0) {
        // channel c's block length is m1 - cur_base of its history record; the history copy below then reads the widened
        // samples (d_in is the staging block here)
        const r8bgpu_buffer& in = *cv->in;
        launch_to_f64(in.format, in.data, in.interleaved != 0, in.stride, const_cast<double*>(d_in), in_stride, cv->max_len,
                      (int) n_ch, in.scale, st, b->rec.d + 2 * ns * n_ch);
        b->launches++;
    }
    if (refill) refill_launch(b, cnt.data(), bp.data(), st);
    for (size_t i = 0; i < ns; i++)
        launch_stage_ragged(b, i, cnt[ns + i], bp[ns + i], b->rec.d + (ns + i) * n_ch, d_in, in_stride, d_out, out_stride, st);
    if (cv != nullptr && cv->out != nullptr && cv->max_count > 0) {
        // channel c's count is e1 - e0 of the last stage's record
        const r8bgpu_buffer& out = *cv->out;
        launch_from_f64(out.format, out.data, out.interleaved != 0, out.stride, d_out, out_stride, cv->max_count, (int) n_ch,
                        out.scale, st, b->rec.d + (2 * ns - 1) * n_ch);
        b->launches++;
    }
    if (tail > 0) {
        launch_save_tail_ragged(d_in, (long long) in_stride, tail, b->dev[0].ring, b->dev[0].ring_cap, b->dev[0].ring_cap - 1,
                                (int) n_ch, st, b->rec.d + 2 * ns * n_ch);
        b->launches++;
    }
    return true;
}

} // extern "C"

// The lock-step calls return one count for every channel; the channels of a mixed batch run different plans.
static bool refuse_mixed_lockstep(const r8bgpu_batch* b, const char* what)
{
    if (b == nullptr || !b->mixed) return false;
    set_err(std::string(what) + ": the channels of a mixed batch run different plans and produce different counts; use "
            "the ragged calls (r8bgpu_batch_process_ragged / _host_ragged / _ragged_fmt / _host_ragged_fmt)");
    return true;
}

// Device buffers live on one GPU: a multi-device batch takes them through its shards.
static bool refuse_front_device(const r8bgpu_batch* b, const char* what)
{
    if (!b->front) return false;
    set_err(std::string(what) + ": device buffers live on one GPU; call the shards of a multi-device batch (r8bgpu_batch_shard())");
    return true;
}

// ---- staging shared by the host path and the sample-format paths ----------------------------

// Samples per row of a staging block for up to n outputs per channel: rows stay 32-byte aligned.
static size_t staging_out_cap(int n) { return ((size_t) n + 3) & ~(size_t) 3; }

static bool ensure_staging(r8bgpu_batch* b)
{
    if (b->st_in != nullptr) return true;
    const Plan& P = *b->plan;
    const size_t in_cap = (size_t) P.max_in_len;
    const size_t o_cap = staging_out_cap(P.max_out_len);
    if (!b->st_in.alloc(b->dev_bytes, in_cap * b->n_ch, "staging: cudaMalloc(in)")) return false;
    if (!b->st_out.alloc(b->dev_bytes, o_cap * b->n_ch, "staging: cudaMalloc(out)")) return false;
    for (Stream* s : {&b->s_h2d, &b->s_d2h, &b->s_comp})
        if (!cuda_ok(cudaStreamCreateWithFlags(s->put(), cudaStreamNonBlocking), "staging: stream")) return false;
    int groups = 8;
    if (const char* e = getenv("R8BGPU_HOST_GROUPS")) groups = atoi(e);
    if (groups < 1) groups = 1;
    while (groups > 1 && b->n_ch / groups < 32) groups /= 2; // keep every group a full-GPU launch
    b->host_groups = groups;
    b->ev_h2d.resize((size_t) groups);
    b->ev_k.resize((size_t) groups);
    for (int i = 0; i < groups; i++)
        if (!cuda_ok(cudaEventCreateWithFlags(b->ev_h2d[(size_t) i].put(), cudaEventDisableTiming), "staging: event") ||
            !cuda_ok(cudaEventCreateWithFlags(b->ev_k[(size_t) i].put(), cudaEventDisableTiming), "staging: event"))
            return false;
    return true;
}

// Device blocks of typed samples as they cross PCIe, 8 bytes per sample of staging room (any format, either layout).
static bool ensure_raw_staging(r8bgpu_batch* b, bool need_in, bool need_out)
{
    const size_t in_cap = (size_t) b->plan->max_in_len;
    const size_t o_cap = staging_out_cap(b->plan->max_out_len);
    return (!need_in || b->raw_in.grow(b->dev_bytes, in_cap * b->n_ch * 8, "process_host: cudaMalloc(raw in)")) &&
           (!need_out || b->raw_out.grow(b->dev_bytes, o_cap * b->n_ch * 8, "process_host: cudaMalloc(raw out)"));
}

static bool buffer_is_plain(const r8bgpu_buffer& d)
{
    return d.format == R8BGPU_F64 && !d.interleaved && d.scale == 1.0;
}

// Whether the chain's first kernel reads the caller's typed input block as it is, instead of a conversion launch widening
// it into the fp64 staging block first: the v2 fused kernel for the wide and one-byte formats (fuses_input_format), the
// half-band decimators (k_hbdown_cascade, k_hbdown) for planar DSD.
static bool input_read_in_kernel(const r8bgpu_batch* b, const r8bgpu_buffer& in)
{
    if (buffer_is_plain(in) || in.interleaved) return false;
    if (!is_dsd_format(in.format)) return fuses_input_format(b);
    return !b->plan->passthrough && !b->dev.empty() && b->plan->stages[0].kind == ST_HBDOWN && !getenv("R8BGPU_NO_FORMAT_FUSION");
}

static r8bgpu_buffer plain_buffer(const double* p, size_t stride)
{
    return r8bgpu_buffer{const_cast<double*>(p), R8BGPU_F64, 0, stride, 1.0};
}

// Host samples of a ragged call cross PCIe as they are into the device block dst (strides count elements, lengths
// samples: format_elem).  Planar: rows 0 .. n-2 as one copy of min(max(lens), stride) elements (reading a row past its
// length stays inside the caller's buffer: the next row starts a stride further on), the last row with its own length,
// dst_stride elements apart; interleaved: the frames of max(lens) samples of the n_ch columns, compact.
static bool h2d_ragged(const r8bgpu_buffer& in, const int* lens, int n_ch, void* dst, size_t dst_stride, cudaStream_t st,
                       const char* what)
{
    const FormatElem fe = format_elem(in.format);
    const size_t e = (size_t) fe.bytes, n = (size_t) n_ch;
    const unsigned char* h = (const unsigned char*) in.data;
    unsigned char* d = (unsigned char*) dst;
    auto ok = [&](cudaError_t err) { return err == cudaSuccess || cuda_ok(err, (std::string(what) + ": H2D").c_str()); };
    int max_len = 0;
    for (int c = 0; c < n_ch; c++) max_len = std::max(max_len, lens[c]);
    if (in.interleaved)
        return max_len == 0 ||
               ok(cudaMemcpy2DAsync(d, n * e, h, in.stride * e, n * e, fe.elems(max_len), cudaMemcpyHostToDevice, st));
    const size_t w = std::min(fe.elems(max_len), in.stride);
    if (n > 1 && w > 0 && !ok(cudaMemcpy2DAsync(d, dst_stride * e, h, in.stride * e, w * e, n - 1, cudaMemcpyHostToDevice, st)))
        return false;
    return lens[n - 1] <= 0 || ok(cudaMemcpyAsync(d + (n - 1) * dst_stride * e, h + (n - 1) * in.stride * e,
                                                  fe.span(lens[n - 1]), cudaMemcpyHostToDevice, st));
}

// Each run of consecutive channels with equal counts goes from the device view dv into the host buffer out as one 2-D
// copy (planar: count samples of the run's rows; interleaved: count frames of the run's columns), so nothing past a
// channel's count is written.
static bool d2h_runs(const r8bgpu_buffer& out, const r8bgpu_buffer& dv, const std::vector<int>& counts, cudaStream_t st,
                     const char* what)
{
    const size_t e = (size_t) format_elem(out.format).bytes, n_ch = counts.size(); // outputs: one sample per element
    unsigned char* h = (unsigned char*) out.data;
    const unsigned char* d = (const unsigned char*) dv.data;
    for (size_t c0 = 0; c0 < n_ch;) {
        size_t c1 = c0 + 1;
        while (c1 < n_ch && counts[c1] == counts[c0]) c1++;
        const size_t k = (size_t) counts[c0], nr = c1 - c0;
        if (k > 0) {
            const cudaError_t err =
                out.interleaved
                    ? cudaMemcpy2DAsync(h + c0 * e, out.stride * e, d + c0 * e, dv.stride * e, nr * e, k, cudaMemcpyDeviceToHost, st)
                    : cudaMemcpy2DAsync(h + c0 * out.stride * e, out.stride * e, d + c0 * dv.stride * e, dv.stride * e, k * e, nr,
                                        cudaMemcpyDeviceToHost, st);
            if (err != cudaSuccess) return cuda_ok(err, (std::string(what) + ": D2H").c_str());
        }
        c0 = c1;
    }
    return true;
}

// The input's lengths (a lock-step call's l, or a ragged call's lens) in whole elements: multiples of 8 for DSD.
static bool check_lengths(const r8bgpu_buffer& in, const int* lens, int n, const char* what)
{
    const int k = format_elem(in.format).samples;
    for (int c = 0; lens != nullptr && c < n; c++)
        if (lens[c] % k != 0) {
            set_err(std::string(what) + ": lengths of a DSD input must be multiples of 8 samples");
            return false;
        }
    return true;
}

static bool check_buffer(const r8bgpu_batch* b, const r8bgpu_buffer* d, const char* what, bool output = false)
{
    if (d == nullptr || format_elem(d->format).bytes == 0) {
        set_err(std::string(what) + ": unknown sample format");
        return false;
    }
    if (output && is_dsd_format(d->format) && !dsd_on(b)) { // a one-bit output runs through the batch's modulators (K8)
        set_err(std::string(what) + ": DSD formats are input-only");
        return false;
    }
    if (d->interleaved && d->stride < (size_t) b->n_ch) {
        set_err(std::string(what) + ": interleaved stride smaller than the channel count");
        return false;
    }
    if (!(d->scale == d->scale) || d->scale == 0.0) {
        set_err(std::string(what) + ": scale must be a non-zero number");
        return false;
    }
    return true;
}

// The part of a caller's buffer that holds channels c0.. (a shard's range): planar rows c0.., or interleaved columns c0..
static r8bgpu_buffer shard_view(const r8bgpu_buffer& d, int c0)
{
    r8bgpu_buffer v = d;
    if (d.data != nullptr) {
        const size_t e = (size_t) format_elem(d.format).bytes;
        v.data = (unsigned char*) d.data + (d.interleaved ? (size_t) c0 * e : (size_t) c0 * d.stride * e);
    }
    return v;
}

// ---- lock-step calls: every channel takes l samples and returns the same count -------------------------------------

// A lock-step call on a batch whose channels diverged runs through the ragged chain, which takes plain buffers only.
static const char* kDivergedTyped =
    "this batch's channels have diverged (ragged calls or clear_channels); typed buffers need channels in lock-step "
    "(clear the batch)";

// Checks a lock-step call of l samples per channel and, while the channels are in lock-step, schedules it into b->calls
// (a passthrough plan has nothing to schedule) and checks the output capacity.  Returns the call's count, or -1 with
// nothing changed.  A batch whose channels diverged is left as it is (returns 0): the caller runs the call through the
// ragged chain, which plans it per group.  saved: the schedule before the call.  Every failure after this puts it back,
// so that a failed call did not happen.
static int schedule_lockstep(r8bgpu_batch* b, const char* what, int l, bool have_in, bool have_out, int out_cap,
                             Schedule& saved)
{
    const std::string w(what);
    if (l < 0 || l > b->plan->max_in_len) {
        set_err(w + ": l must be in [0, MaxInLen]");
        return -1;
    }
    if (l > 0 && !have_in) {
        set_err(w + ": null input");
        return -1;
    }
    saved = b->sched;
    if (b->diverged) return 0;
    if (b->plan->passthrough) { // SrcSampleRate == DstSampleRate: the reference hands the input back
        if (l <= out_cap) return l;
        set_err(w + ": output capacity too small");
        return -1;
    }
    const int n = b->sched.advance(l, b->calls);
    if (n > out_cap || (n > 0 && !have_out)) {
        b->sched = saved;
        set_err(w + ": output capacity too small for this call");
        return -1;
    }
    return n;
}

// Queues one lock-step call (scheduled in b->calls: l samples in, n out per channel) for channels [ch0, ch0 + nch) on
// st.  in / out are device views whose channel 0 is channel ch0: the caller's buffers, or a host call's staging rows.
// A typed side is read or written by the chain's first / last kernel itself where it can, else converted through the
// fp64 staging rows of these channels.  dh: this call's dither records (nullptr: no channel dithers), filled here for
// these channels; n0: each channel's output total before the call.
static bool launch_lockstep(r8bgpu_batch* b, const r8bgpu_buffer& in, const r8bgpu_buffer& out, int l, int n, int ch0,
                            int nch, cudaStream_t st, DitherRec* dh, const std::vector<long long>& n0)
{
    const size_t in_cap = (size_t) b->plan->max_in_len;
    const size_t o_cap = staging_out_cap(b->plan->max_out_len);
    const bool in_plain = buffer_is_plain(in), out_plain = buffer_is_plain(out);
    const bool in_fused = input_read_in_kernel(b, in);
    // flat TPDF runs in the fused kernel's stores; a call with a shaped channel converts through k_dither_shape
    const bool out_fused = !out_plain && !out.interleaved && fuses_output_format(b) && !(dh && dither_shaped(b, ch0, nch));
    TypedIO tio;
    if (dh != nullptr) {
        for (int c = ch0; c < ch0 + nch; c++) dh[c] = DitherRec{b->st_out + (size_t) c * o_cap, n, n0[(size_t) c], 0};
        if (out_fused) {
            long long mf = 0, ms = 0;
            if (!dither_upload(b, ch0, nch, st, mf, ms)) return false;
            tio.out_dither = b->dith->d_call;
        }
    }
    const double* src = (const double*) in.data;
    size_t src_stride = in.stride;
    if (in_fused) { // the first kernel reads the caller's samples as they are
        tio.in_fmt = in.format;
        tio.in_scale = in.scale;
    } else if (!in_plain) {
        double* wide = b->st_in + (size_t) ch0 * in_cap;
        launch_to_f64(in.format, in.data, in.interleaved != 0, in.stride, wide, in_cap, l, nch, in.scale, st);
        if (l > 0) b->launches++;
        src = wide;
        src_stride = in_cap;
    }
    double* dst = (double*) out.data;
    size_t dst_stride = out.stride;
    if (out_fused) { // the last kernel narrows in its stores
        tio.out_fmt = out.format;
        tio.out_scale = out.scale;
    } else if (!out_plain) {
        dst = b->st_out + (size_t) ch0 * o_cap;
        dst_stride = o_cap;
    }
    if (b->plan->passthrough) {
        if (l > 0 && !cuda_ok(cudaMemcpy2DAsync(dst, dst_stride * sizeof(double), src, src_stride * sizeof(double),
                                                (size_t) l * sizeof(double), (size_t) nch, cudaMemcpyDeviceToDevice, st),
                              "passthrough copy"))
            return false;
    } else {
        launch_call(b, b->calls, src, src_stride, l, dst, dst_stride, ch0, nch, st, tio);
    }
    if (!out_plain && !out_fused) {
        launch_from_f64(out.format, out.data, out.interleaved != 0, out.stride, dst, o_cap, n, nch, out.scale, st);
        if (n > 0) b->launches++;
    }
    return dh == nullptr || out_fused || dither_launch(b, out, ch0, nch, st);
}

// ---- channels with schedules of their own, buffers of any format -----------------------------
// One conversion pass in front of the per-stage chain and one behind it, through the fp64 staging blocks.  A plain side
// (planar F64, scale 1) is read or written by the chain itself.

// Queues a call planned in `step` on st; in / out are device buffers, lens the block lengths.
static bool launch_ragged_fmt(r8bgpu_batch* b, const RaggedSchedule::Step& step, const int* lens, const r8bgpu_buffer& in,
                              const r8bgpu_buffer& out, cudaStream_t st)
{
    const Plan& P = *b->plan;
    const int n_ch = b->n_ch;
    const size_t in_cap = (size_t) P.max_in_len;
    const size_t o_cap = staging_out_cap(P.max_out_len);
    const bool in_plain = buffer_is_plain(in), out_plain = buffer_is_plain(out);
    RaggedConv cv;
    cv.in = in_plain ? nullptr : &in;
    cv.out = out_plain ? nullptr : &out;
    for (int c = 0; c < n_ch; c++) {
        cv.max_len = std::max(cv.max_len, lens[c]);
        cv.max_count = std::max(cv.max_count, step.count[(size_t) step.key_of[(size_t) c]]);
    }
    const double* x = in_plain ? (const double*) in.data : b->st_in;
    size_t xs = in_plain ? in.stride : in_cap;
    // dithered channels: their outputs are re-quantised from the fp64 rows once the usual conversion has run
    const bool dith = dither_active(b, out.format, 0, n_ch);
    const std::vector<long long> n0 = dith ? outputs_before(b) : std::vector<long long>();
    auto dither_out = [&](const double* rows, size_t stride, bool by_len) {
        if (!dith) return true;
        DitherRec* h = dither_records(b);
        if (h == nullptr) return false;
        for (int c = 0; c < n_ch; c++)
            h[c] = DitherRec{rows + (size_t) c * stride, by_len ? lens[c] : step.count[(size_t) step.key_of[(size_t) c]],
                             n0[(size_t) c]};
        return dither_launch(b, out, 0, n_ch, st);
    };
    if (!P.passthrough)
        return launch_ragged(b, b->rag, step, x, xs, out_plain ? (double*) out.data : b->st_out, out_plain ? out.stride : o_cap,
                             st, &cv) &&
               dither_out(b->st_out, o_cap, false);
    if (in_plain && out_plain) { // passthrough: one copy per run of channels with one block length, nothing past lens[c]
        for (const RaggedSchedule::Run& r : step.runs) {
            const int l = step.len[(size_t) r.key];
            if (l > 0 && !cuda_ok(cudaMemcpy2DAsync((double*) out.data + (size_t) r.c0 * out.stride, out.stride * sizeof(double),
                                                    x + (size_t) r.c0 * xs, xs * sizeof(double), (size_t) l * sizeof(double),
                                                    (size_t) r.n, cudaMemcpyDeviceToDevice, st),
                                  "batch_process_ragged: passthrough copy"))
                return false;
        }
        return true;
    }
    // passthrough: there are no stage records, so each channel's extent (its block length, which is also its count) goes
    // up in a record of its own
    if (!ensure_ragged_state(b)) return false;
    RaggedRec* h = b->rec.next("ragged: records");
    if (h == nullptr) return false;
    for (int c = 0; c < n_ch; c++) {
        memset(&h[c], 0, sizeof h[c]);
        h[c].m1 = h[c].e1 = lens[c];
    }
    if (!b->rec.upload(0, (size_t) n_ch, st, "ragged: record upload")) return false;
    if (cv.max_len == 0) return true;
    if (!in_plain) { // widened straight into a plain output, else into the staging block
        double* dst = out_plain ? (double*) out.data : b->st_in;
        xs = out_plain ? out.stride : in_cap;
        launch_to_f64(in.format, in.data, in.interleaved != 0, in.stride, dst, xs, cv.max_len, n_ch, in.scale, st, b->rec.d);
        b->launches++;
        x = dst;
    }
    if (!out_plain) {
        launch_from_f64(out.format, out.data, out.interleaved != 0, out.stride, x, xs, cv.max_len, n_ch, out.scale, st, b->rec.d);
        b->launches++;
    }
    return dither_out(x, xs, true);
}

// Device buffers; asynchronous on the batch stream.  A call with plain buffers on both sides allocates no staging.
// lockstep: a lock-step call on a batch whose channels diverged -- returns their common count (else 0).
static int process_ragged_dev(r8bgpu_batch* b, const r8bgpu_buffer& in, const int* lens, const r8bgpu_buffer& out,
                              int out_cap, int* counts, bool lockstep)
{
    const bool plain = buffer_is_plain(in) && buffer_is_plain(out);
    const std::string what = plain ? "batch_process_ragged" : "batch_process_ragged_fmt";
    DeviceGuard g(b->device);
    RaggedSchedule::Step step;
    if (!plan_ragged(b, what.c_str(), lens, in.data != nullptr, out.data != nullptr, out_cap, lockstep, step)) return -1;
    if (!plain && !ensure_staging(b)) return -1;
    if (!launch_ragged_fmt(b, step, lens, in, out, b->stream)) return -1;
    if (!cuda_ok(cudaGetLastError(), (what + ": kernel launch").c_str())) return -1;
    if (counts != nullptr)
        for (int c = 0; c < b->n_ch; c++) counts[c] = step.count[(size_t) step.key_of[(size_t) c]];
    const int common = step.count.empty() ? 0 : step.count[0];
    adopt_step(b, step);
    return lockstep ? common : 0;
}

// Host buffers: the narrow samples cross PCIe as they are (h2d_ragged), the device converts them, runs the chain and
// converts back, and each run of consecutive channels with equal counts comes back as one 2-D block (d2h_runs).
// Synchronises.  lockstep: as in process_ragged_dev.
static int process_host_ragged_fmt_impl(r8bgpu_batch* b, const r8bgpu_buffer& in, const int* lens, const r8bgpu_buffer& out,
                                        int out_cap, int* counts, bool lockstep)
{
    const bool in_plain = buffer_is_plain(in), out_plain = buffer_is_plain(out);
    const std::string what = in_plain && out_plain ? "batch_process_host_ragged" : "batch_process_host_ragged_fmt";
    if (b->front) {
        if (lens == nullptr) {
            set_err(what + ": null lens");
            return -1;
        }
        const ShardFront& F = *b->front;
        return front_call(
            b,
            [&](r8bgpu_batch* sb, int s) {
                RaggedSchedule::Step dry;
                return plan_ragged(sb, what.c_str(), lens + F.ch0[(size_t) s], in.data != nullptr, out.data != nullptr, out_cap,
                                   lockstep, dry);
            },
            [&](r8bgpu_batch* sb, int s) {
                const int c0 = F.ch0[(size_t) s];
                return process_host_ragged_fmt_impl(sb, shard_view(in, c0), lens + c0, shard_view(out, c0), out_cap,
                                                    counts != nullptr ? counts + c0 : nullptr, lockstep);
            });
    }
    DeviceGuard g(b->device);
    RaggedSchedule::Step step;
    if (!plan_ragged(b, what.c_str(), lens, in.data != nullptr, out.data != nullptr, out_cap, lockstep, step)) return -1;
    if (!ensure_staging(b) || !ensure_raw_staging(b, !in_plain, !out_plain)) return -1;
    // order after any device-path work queued on the batch stream (the two paths share the rings and the staging)
    if (!cuda_ok(cudaStreamSynchronize(b->stream), (what + ": sync(batch stream)").c_str())) return -1;
    const size_t in_cap = (size_t) b->plan->max_in_len;
    const size_t o_cap = staging_out_cap(b->plan->max_out_len);
    const cudaStream_t st = b->s_comp;
    const int n_ch = b->n_ch;
    std::vector<int> cnt((size_t) n_ch);
    for (int c = 0; c < n_ch; c++) cnt[(size_t) c] = step.count[(size_t) step.key_of[(size_t) c]];
    unsigned char* din = in_plain ? (unsigned char*) (double*) b->st_in : b->raw_in;
    unsigned char* dout = out_plain ? (unsigned char*) (double*) b->st_out : b->raw_out;
    // device copies: planar [n_ch][in_cap] / [n_ch][o_cap], interleaved compact [frames][n_ch]
    const r8bgpu_buffer dv_in = {din, in.format, in.interleaved, in.interleaved ? (size_t) n_ch : in_cap, in.scale};
    // a plain passthrough call launches nothing: its output is the input staging rows
    const bool copy_only = b->plan->passthrough && in_plain && out_plain;
    const r8bgpu_buffer dv_out = copy_only ? dv_in
                                           : r8bgpu_buffer{dout, out.format, out.interleaved,
                                                           out.interleaved ? (size_t) n_ch : o_cap, out.scale};
    bool ok = h2d_ragged(in, lens, n_ch, din, in_cap, st, what.c_str());
    ok = ok && (copy_only || launch_ragged_fmt(b, step, lens, dv_in, dv_out, st));
    ok = ok && d2h_runs(out, dv_out, cnt, st, what.c_str());
    ok = cuda_ok(cudaStreamSynchronize(st), (what + ": sync").c_str()) && ok;
    if (!ok || !cuda_ok(cudaGetLastError(), (what + ": kernel launch").c_str())) return -1;
    if (counts != nullptr)
        for (int c = 0; c < n_ch; c++) counts[c] = cnt[(size_t) c];
    const int common = step.count.empty() ? 0 : step.count[0];
    adopt_step(b, step);
    return lockstep ? common : 0;
}

// Device buffers of any format, channels in lock-step; asynchronous on the batch stream.  A call with plain buffers on
// both sides allocates no staging.
static int process_dev(r8bgpu_batch* b, const char* what, const r8bgpu_buffer& in, int l, const r8bgpu_buffer& out,
                       int out_cap)
{
    const bool plain = buffer_is_plain(in) && buffer_is_plain(out);
    const bool dith = dither_active(b, out.format, 0, b->n_ch);
    const std::vector<long long> n0 = dith ? outputs_before(b) : std::vector<long long>();
    Schedule saved;
    const int n = schedule_lockstep(b, what, l, in.data != nullptr, out.data != nullptr, out_cap, saved);
    if (n < 0) return -1;
    if (b->diverged) {
        if (!plain) {
            set_err(std::string(what) + ": " + kDivergedTyped);
            return -1;
        }
        const std::vector<int> lens((size_t) b->n_ch, l);
        return process_ragged_dev(b, in, lens.data(), out, out_cap, nullptr, true);
    }
    DeviceGuard g(b->device);
    const cudaStream_t st = b->stream;
    DitherRec* dh = nullptr;
    if ((plain || ensure_staging(b)) && (!dith || (dh = dither_records(b)) != nullptr) && upload_fasttiming(b, st) &&
        launch_lockstep(b, in, out, l, n, 0, b->n_ch, st, dh, n0) &&
        cuda_ok(cudaGetLastError(), (std::string(what) + ": kernel launch").c_str())) {
        count_passthrough(b, l);
        return n;
    }
    b->sched = saved; // a failed call did not happen
    return -1;
}

// Host-pointer path.  The batch is cut into channel groups that flow through a three-stage pipeline
//   copy stream A: H2D(group g+1)  |  compute stream: kernels(group g)  |  copy stream B: D2H(group g-1)
// so the two PCIe directions and the SMs work at the same time (channels are independent, so a group
// is a self-contained sub-batch).  Staging buffers are per channel, so groups never alias.
// Narrow / interleaved sample formats cross PCIe as they are and are widened (narrowed) on the
// device by r8b_format.cu, in the compute stage of the same pipeline.
static int process_host_impl(r8bgpu_batch* b, const r8bgpu_buffer& in, int l, const r8bgpu_buffer& out, int out_cap)
{
    if (refuse_mixed_lockstep(b, "batch_process_host")) return -1;
    const bool in_plain = buffer_is_plain(in), out_plain = buffer_is_plain(out);
    if (b->front) {
        const ShardFront& F = *b->front;
        long long common = -1; // every shard must also produce the same count
        return front_call(
            b,
            [&](r8bgpu_batch* sb, int) {
                if (b->plan->passthrough || l < 0 || l > b->plan->max_in_len) return true; // (the shards refuse such an l)
                int n = 0;
                if (sb->diverged) {
                    if (!in_plain || !out_plain) {
                        set_err(std::string("batch_process_host_fmt: ") + kDivergedTyped);
                        return false;
                    }
                    const std::vector<int> lens((size_t) sb->n_ch, l);
                    RaggedSchedule::Step dry;
                    if (!plan_ragged(sb, "batch_process_host", lens.data(), in.data != nullptr, out.data != nullptr, out_cap,
                                     true, dry))
                        return false;
                    n = dry.count.empty() ? 0 : dry.count[0];
                } else {
                    Schedule t = sb->sched;
                    std::vector<StageCall> c;
                    n = t.advance(l, c);
                }
                if (common >= 0 && n != common) {
                    set_err("batch_process_host: this batch's channels have diverged (ragged calls or clear_channels) and "
                            "would produce " + std::to_string(common) + " and " + std::to_string(n) +
                            " samples; use r8bgpu_batch_process_host_ragged, or clear the batch");
                    return false;
                }
                common = n;
                return true;
            },
            [&](r8bgpu_batch* sb, int s) {
                return process_host_impl(sb, shard_view(in, F.ch0[(size_t) s]), l, shard_view(out, F.ch0[(size_t) s]),
                                         out_cap);
            });
    }
    const bool dith = dither_active(b, out.format, 0, b->n_ch);
    const std::vector<long long> n0 = dith ? outputs_before(b) : std::vector<long long>();
    Schedule saved;
    const int n = schedule_lockstep(b, "batch_process_host", l, in.data != nullptr, out.data != nullptr, out_cap, saved);
    if (n < 0) return -1;
    if (b->diverged) {
        if (!in_plain || !out_plain) {
            set_err(std::string("batch_process_host_fmt: ") + kDivergedTyped);
            return -1;
        }
        const std::vector<int> lens((size_t) b->n_ch, l);
        return process_host_ragged_fmt_impl(b, in, lens.data(), out, out_cap, nullptr, true);
    }
    DeviceGuard g(b->device);
    DitherRec* dh = nullptr;
    if (!ensure_staging(b) || !ensure_raw_staging(b, !in_plain, !out_plain) || (dith && (dh = dither_records(b)) == nullptr)) {
        b->sched = saved;
        return -1;
    }
    // any failure from here on: put the schedule back and drain the pipeline streams, so that the rings and the schedule
    // still agree on the next call (the failed call then simply did not happen)
    auto fail = [&]() {
        b->sched = saved;
        cudaStreamSynchronize(b->s_h2d);
        cudaStreamSynchronize(b->s_comp);
        cudaStreamSynchronize(b->s_d2h);
        return -1;
    };
    // order after any device-path work queued on the batch stream (the two paths share the rings)
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "process_host: sync(batch stream)")) return fail();
    if (!upload_fasttiming(b, b->s_comp)) return fail();
    const size_t in_cap = (size_t) b->plan->max_in_len;
    const size_t o_cap = staging_out_cap(b->plan->max_out_len);
    const FormatElem fin = format_elem(in.format);
    const size_t ein = (size_t) fin.bytes;
    const int G = b->host_groups;
    const unsigned char* hin = (const unsigned char*) in.data;
    for (int gi = 0; gi < G; gi++) {
        const int ch0 = (int) ((long long) b->n_ch * gi / G);
        const int ch1 = (int) ((long long) b->n_ch * (gi + 1) / G);
        const int nch = ch1 - ch0;
        if (nch <= 0) continue;
        double* din = b->st_in + (size_t) ch0 * in_cap;
        double* dout = b->st_out + (size_t) ch0 * o_cap;
        unsigned char* rin = in_plain ? nullptr : b->raw_in + (size_t) ch0 * in_cap * 8;
        unsigned char* rout = out_plain ? nullptr : b->raw_out + (size_t) ch0 * o_cap * 8;
        if (l > 0) {
            cudaError_t e;
            if (in_plain)
                e = cudaMemcpy2DAsync(din, in_cap * 8, hin + (size_t) ch0 * in.stride * 8, in.stride * 8,
                                      (size_t) l * 8, (size_t) nch, cudaMemcpyHostToDevice, b->s_h2d);
            else if (in.interleaved) // device copy: compact [frames of l samples][nch]
                e = cudaMemcpy2DAsync(rin, (size_t) nch * ein, hin + (size_t) ch0 * ein, in.stride * ein,
                                      (size_t) nch * ein, fin.elems(l), cudaMemcpyHostToDevice, b->s_h2d);
            else // device copy: [nch][in_cap elements]
                e = cudaMemcpy2DAsync(rin, in_cap * ein, hin + (size_t) ch0 * in.stride * ein, in.stride * ein,
                                      fin.span(l), (size_t) nch, cudaMemcpyHostToDevice, b->s_h2d);
            if (!cuda_ok(e, "process_host: H2D")) return fail();
        }
        cudaEventRecord(b->ev_h2d[(size_t) gi], b->s_h2d);
        cudaStreamWaitEvent(b->s_comp, b->ev_h2d[(size_t) gi], 0);
        const r8bgpu_buffer vin = in_plain ? plain_buffer(din, in_cap)
                                           : r8bgpu_buffer{rin, in.format, in.interleaved,
                                                           in.interleaved ? (size_t) nch : in_cap, in.scale};
        const r8bgpu_buffer vout = out_plain ? plain_buffer(dout, o_cap)
                                             : r8bgpu_buffer{rout, out.format, out.interleaved,
                                                             out.interleaved ? (size_t) nch : o_cap, out.scale};
        if (!launch_lockstep(b, vin, vout, l, n, ch0, nch, b->s_comp, dh, n0)) return fail();
        cudaEventRecord(b->ev_k[(size_t) gi], b->s_comp);
        cudaStreamWaitEvent(b->s_d2h, b->ev_k[(size_t) gi], 0);
        // every channel of the group has n samples: one 2-D copy
        if (!d2h_runs(shard_view(out, ch0), vout, std::vector<int>((size_t) nch, n), b->s_d2h, "process_host")) return fail();
    }
    if (!cuda_ok(cudaStreamSynchronize(b->s_d2h), "process_host: sync")) return fail();
    if (!cuda_ok(cudaStreamSynchronize(b->s_comp), "process_host: sync")) return fail();
    if (!cuda_ok(cudaGetLastError(), "process_host: kernel launch")) return fail();
    count_passthrough(b, l);
    return n;
}

extern "C" {

int r8bgpu_batch_process(r8bgpu_batch* b, const double* d_in, size_t in_stride, int l, double* d_out,
                         size_t out_stride, int out_cap)
{
    if (refuse_mixed_lockstep(b, "batch_process")) return -1;
    if (b == nullptr) {
        set_err("batch_process: null batch");
        return -1;
    }
    if (refuse_dsd_plain(b, "batch_process")) return -1;
    if (refuse_front_device(b, "batch_process")) return -1;
    return process_dev(b, "batch_process", plain_buffer(d_in, in_stride), l, plain_buffer(d_out, out_stride), out_cap);
}

// mixed batches (below, after the flush helpers they share)
static int mixed_ragged(r8bgpu_batch* b, const char* what, const r8bgpu_buffer& in, const int* lens, const r8bgpu_buffer& out,
                        int out_cap, int* counts, bool host);
static int mixed_flush(r8bgpu_batch* b, const char* what, const int* channels, int n, const long long* targets,
                       const r8bgpu_buffer& out, int out_cap, int* counts, bool host);
// one-bit DSD output (below)
static int dsd_process(r8bgpu_batch* b, const char* what, const r8bgpu_buffer& in, int l, const int* lens,
                       const r8bgpu_buffer& out, int out_cap, int* counts, bool host);
static int dsd_flush(r8bgpu_batch* b, const char* what, const int* channels, int n, const long long* targets,
                     const r8bgpu_buffer& out, int out_cap, int* counts, bool host);

int r8bgpu_batch_process_ragged(r8bgpu_batch* b, const double* d_in, size_t in_stride, const int* lens, double* d_out,
                                size_t out_stride, int out_cap, int* counts)
{
    if (b == nullptr || counts == nullptr) {
        set_err("batch_process_ragged: null batch or counts");
        return -1;
    }
    if (refuse_dsd_plain(b, "batch_process_ragged")) return -1;
    const r8bgpu_buffer in = plain_buffer(d_in, in_stride), out = plain_buffer(d_out, out_stride);
    if (b->mixed) return mixed_ragged(b, "batch_process_ragged", in, lens, out, out_cap, counts, false);
    if (refuse_front_device(b, "batch_process_ragged")) return -1;
    return process_ragged_dev(b, in, lens, out, out_cap, counts, false);
}

int r8bgpu_batch_process_host_ragged(r8bgpu_batch* b, const double* h_in, size_t in_stride, const int* lens, double* h_out,
                                     size_t out_stride, int out_cap, int* counts)
{
    if (b == nullptr || counts == nullptr) {
        set_err("batch_process_host_ragged: null batch or counts");
        return -1;
    }
    if (refuse_dsd_plain(b, "batch_process_host_ragged")) return -1;
    const r8bgpu_buffer in = plain_buffer(h_in, in_stride), out = plain_buffer(h_out, out_stride);
    if (b->mixed) return mixed_ragged(b, "batch_process_host_ragged", in, lens, out, out_cap, counts, true);
    return process_host_ragged_fmt_impl(b, in, lens, out, out_cap, counts, false);
}

// Typed device buffers; asynchronous on the batch stream.
int r8bgpu_batch_process_ragged_fmt(r8bgpu_batch* b, const r8bgpu_buffer* d_in, const int* lens, const r8bgpu_buffer* d_out,
                                    int out_cap, int* counts)
{
    if (b == nullptr || counts == nullptr) {
        set_err("batch_process_ragged_fmt: null batch or counts");
        return -1;
    }
    if (refuse_front_device(b, "batch_process_ragged_fmt")) return -1;
    if (!check_buffer(b, d_in, "batch_process_ragged_fmt(in)") || !check_buffer(b, d_out, "batch_process_ragged_fmt(out)", true) ||
        !check_lengths(*d_in, lens, b->n_ch, "batch_process_ragged_fmt"))
        return -1;
    if (dsd_on(b)) {
        if (lens == nullptr) {
            set_err("batch_process_ragged_fmt: null lens");
            return -1;
        }
        return dsd_process(b, "batch_process_ragged_fmt", *d_in, 0, lens, *d_out, out_cap, counts, false);
    }
    if (b->mixed) return mixed_ragged(b, "batch_process_ragged_fmt", *d_in, lens, *d_out, out_cap, counts, false);
    return process_ragged_dev(b, *d_in, lens, *d_out, out_cap, counts, false);
}

int r8bgpu_batch_process_host_ragged_fmt(r8bgpu_batch* b, const r8bgpu_buffer* h_in, const int* lens, const r8bgpu_buffer* h_out,
                                         int out_cap, int* counts)
{
    if (b == nullptr || counts == nullptr) {
        set_err("batch_process_host_ragged_fmt: null batch or counts");
        return -1;
    }
    if (!check_buffer(b, h_in, "batch_process_host_ragged_fmt(in)") ||
        !check_buffer(b, h_out, "batch_process_host_ragged_fmt(out)", true) ||
        !check_lengths(*h_in, lens, b->n_ch, "batch_process_host_ragged_fmt"))
        return -1;
    if (dsd_on(b)) {
        if (lens == nullptr) {
            set_err("batch_process_host_ragged_fmt: null lens");
            return -1;
        }
        return dsd_process(b, "batch_process_host_ragged_fmt", *h_in, 0, lens, *h_out, out_cap, counts, true);
    }
    if (b->mixed) return mixed_ragged(b, "batch_process_host_ragged_fmt", *h_in, lens, *h_out, out_cap, counts, true);
    return process_host_ragged_fmt_impl(b, *h_in, lens, *h_out, out_cap, counts, false);
}

int r8bgpu_batch_clear_channels(r8bgpu_batch* b, const int* channels, int n)
{
    if (b == nullptr || n < 0 || (n > 0 && channels == nullptr)) {
        set_err("batch_clear_channels: bad arguments");
        return -1;
    }
    if (!check_channels(b, channels, n, "batch_clear_channels", false)) return -1;
    if (n == 0) return 0;
    if (sub_batches(b)) { // every index is valid: each shard or part clears its own channels
        for (const ChannelGroup& G : group_channels(b, channels, n))
            if (!G.rows.empty() && r8bgpu_batch_clear_channels(G.b, G.rows.data(), (int) G.rows.size()) != 0) return -1;
        if (!b->mixed) return 0;
        // a mixed batch keeps the dither and DSD modulator state of its channels
        DeviceGuard g(b->device);
        if (!dither_clear(b, channels, n, b->stream) || !dsd_clear(b, channels, n, b->stream) ||
            !cuda_ok(cudaStreamSynchronize(b->stream), "batch_clear_channels: sync"))
            return -1;
        return 0;
    }
    if (has_fasttiming(*b->plan)) {
        std::vector<char> named((size_t) b->n_ch, 0);
        int distinct = 0;
        for (int i = 0; i < n; i++) distinct += named[(size_t) channels[i]] ? 0 : (named[(size_t) channels[i]] = 1);
        if (distinct == b->n_ch) return r8bgpu_batch_clear(b);
        set_err("batch_clear_channels: R8B_FASTTIMING plans run lock-step only; clear every channel (r8bgpu_batch_clear)");
        return -1;
    }
    DeviceGuard g(b->device);
    for (const StageDev& d : b->dev) {
        if (d.ring == nullptr) continue;
        for (int i = 0; i < n; i++)
            if (!cuda_ok(cudaMemsetAsync(d.ring + (size_t) channels[i] * (size_t) d.ring_cap, 0, (size_t) d.ring_cap * sizeof(double),
                                         b->stream), "batch_clear_channels: cudaMemsetAsync"))
                return -1;
    }
    if (!dither_clear(b, channels, n, b->stream) || !dsd_clear(b, channels, n, b->stream)) return -1;
    // as r8bgpu_batch_clear(): finished here, so the host path's pipeline streams see the cleared rings
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "batch_clear_channels: sync")) return -1;
    for (int i = 0; i < n; i++) b->pass_n[(size_t) channels[i]] = 0;
    channel_schedules(b);
    b->rag.clear_channels(channels, n);
    b->diverged = !b->rag.converged();
    if (!b->diverged) b->sched = b->rag.groups[0];
    return 0;
}

// ---- per-channel rate trim (trim plans, r8bgpu_plan_create_trim) ------------------------------------------------------

int r8bgpu_batch_set_trim(r8bgpu_batch* b, const int* channels, int n, const double* factors)
{
    if (b == nullptr || n < 0 || (n > 0 && (channels == nullptr || factors == nullptr))) {
        set_err("batch_set_trim: bad arguments");
        return -1;
    }
    // every check before anything changes: a refused call changes nothing
    if (!check_channels(b, channels, n, "batch_set_trim", true, [&](int i, int c) {
            const Plan& P = *slot_of(b, c).b->plan;
            if (P.trim_stage < 0) {
                set_err("batch_set_trim: channel " + std::to_string(c) + " runs a plan that is not a trim plan "
                        "(r8bgpu_plan_create_trim)");
                return false;
            }
            if (!P.trim_factor_ok(factors[i])) {
                char msg[160];
                snprintf(msg, sizeof msg, "batch_set_trim: factor %.17g of channel %d outside [1 - max_trim, 1 + max_trim] "
                         "(max_trim %g)", factors[i], c, P.max_trim);
                set_err(msg);
                return false;
            }
            return true;
        }))
        return -1;
    if (n == 0) return 0;
    if (sub_batches(b)) { // route each channel to its part (mixed) or shard (multi-device)
        for (const ChannelGroup& G : group_channels(b, channels, n))
            if (!G.rows.empty() &&
                r8bgpu_batch_set_trim(G.b, G.rows.data(), (int) G.rows.size(), gather(factors, G.idx).data()) != 0)
                return -1;
        return 0;
    }
    const Plan& P = *b->plan;
    std::vector<double> dsr((size_t) n);
    for (int i = 0; i < n; i++) {
        dsr[(size_t) i] = P.trim_dsr(factors[i]);
        b->trim[(size_t) channels[i]] = factors[i];
    }
    channel_schedules(b);
    b->rag.retime_channels(channels, n, dsr.data());
    b->diverged = !b->rag.converged();
    if (!b->diverged) b->sched = b->rag.groups[0];
    return 0;
}

int r8bgpu_batch_trim(const r8bgpu_batch* b, double* factors)
{
    if (b == nullptr || factors == nullptr) {
        set_err("batch_trim: bad arguments");
        return -1;
    }
    for (int c = 0; c < b->n_ch; c++) {
        const Slot s = slot_of(b, c);
        factors[c] = s.b->trim.empty() ? 1.0 : s.b->trim[(size_t) s.row];
    }
    return 0;
}

// ---- dithered integer output (r8b_dither.cuh) -------------------------------------------------------------------------

int r8bgpu_batch_set_dither(r8bgpu_batch* b, const int* channels, int n, const r8bgpu_dither* cfg)
{
    if (b == nullptr || n < 0 || (n > 0 && (channels == nullptr || cfg == nullptr))) {
        set_err("batch_set_dither: bad arguments");
        return -1;
    }
    // every check before anything changes: a refused call changes nothing
    if (!check_channels(b, channels, n, "batch_set_dither", true, [&](int i, int c) {
            std::string why;
            if (dither_cfg_ok(cfg[i], why)) return true;
            set_err("batch_set_dither: channel " + std::to_string(c) + ": " + why);
            return false;
        }))
        return -1;
    if (n == 0) return 0;
    if (b->front) { // channel ranges go to the shards
        for (const ChannelGroup& G : group_channels(b, channels, n))
            if (!G.rows.empty() &&
                r8bgpu_batch_set_dither(G.b, G.rows.data(), (int) G.rows.size(), gather(cfg, G.idx).data()) != 0)
                return -1;
        return 0;
    }
    // ordinary and mixed batches keep the settings themselves: they own the conversion into the caller's buffer
    DeviceGuard g(b->device);
    const size_t n_ch = (size_t) b->n_ch;
    if (!b->dith) {
        std::unique_ptr<DitherState> D(new DitherState);
        D->cfg.assign(n_ch, DitherCfg{});
        D->m.assign(n_ch, 0);
        if (!D->d_cfg.alloc(b->dev_bytes, n_ch, "batch_set_dither: cudaMalloc") ||
            !D->d_err.alloc(b->dev_bytes, n_ch * kDitherTaps, "batch_set_dither: cudaMalloc") ||
            !D->rec.create(b->dev_bytes, n_ch, "batch_set_dither: cudaMalloc", "batch_set_dither: cudaMallocHost",
                           "batch_set_dither: cudaEventCreate") ||
            !cuda_ok(cudaMemset(D->d_err, 0, n_ch * kDitherTaps * sizeof(double)), "batch_set_dither: cudaMemset") ||
            !D->d_call.upload(b->dev_bytes, {DitherCall{D->d_cfg, D->rec.d, D->d_err}}, "batch_set_dither: cudaMalloc",
                              "batch_set_dither: upload"))
            return -1;
        b->dith = std::move(D);
    }
    DitherState& D = *b->dith;
    // queued calls read the settings they were queued with
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "batch_set_dither: sync")) return -1;
    std::vector<DitherCfg> next = D.cfg;
    for (int i = 0; i < n; i++) {
        DitherCfg d{};
        d.kind = cfg[i].kind;
        d.seed = cfg[i].kind == R8BGPU_DITHER_OFF ? 0 : cfg[i].seed;
        d.n_taps = cfg[i].n_taps;
        for (int k = 0; k < cfg[i].n_taps; k++) d.taps[k] = cfg[i].taps[k];
        next[(size_t) channels[i]] = d;
    }
    if (!cuda_ok(cudaMemcpy(D.d_cfg, next.data(), n_ch * sizeof(DitherCfg), cudaMemcpyHostToDevice), "batch_set_dither: upload"))
        return -1;
    D.cfg.swap(next);
    D.any = false;
    for (const DitherCfg& d : D.cfg) D.any = D.any || d.kind != R8BGPU_DITHER_OFF;
    return 0;
}

int r8bgpu_dither_quantize_host(const r8bgpu_dither* cfg, int fmt, double scale, const double* y, int n, long long first_index,
                                double* err_state, void* out)
{
    if (cfg == nullptr || n < 0 || (n > 0 && (y == nullptr || out == nullptr)) || err_state == nullptr || first_index < 0) {
        set_err("dither_quantize_host: bad arguments");
        return -1;
    }
    std::string why;
    if (!dither_cfg_ok(*cfg, why)) {
        set_err("dither_quantize_host: " + why);
        return -1;
    }
    if (!is_int_format(fmt)) {
        set_err("dither_quantize_host: fmt must be R8BGPU_S16, R8BGPU_S24, R8BGPU_S32, R8BGPU_U8, R8BGPU_ULAW or R8BGPU_ALAW");
        return -1;
    }
    long long lo, hi;
    dither_range(fmt, lo, hi);
    double tap[kDitherTaps] = {}, eh[kDitherTaps] = {};
    const int K = cfg->kind == R8BGPU_DITHER_OFF ? 0 : cfg->n_taps;
    for (int k = 0; k < kDitherTaps; k++) {
        tap[k] = k < K ? cfg->taps[k] : 0.0;
        eh[k] = err_state[k];
    }
    for (int i = 0; i < n; i++) {
        const double v = y[i] * scale;
        long long q;
        if (cfg->kind == R8BGPU_DITHER_OFF) { // the cast: truncation toward zero, saturation, NaN -> 0
            q = v != v ? 0 : (v <= (double) lo ? lo : (v >= (double) hi ? hi : (long long) v));
        } else {
            q = dither_step(tap, K, eh, cfg->seed, first_index + i, v, lo, hi);
        }
        if (fmt == FMT_S16) {
            static_cast<short*>(out)[i] = (short) q;
        } else if (fmt == FMT_S32) {
            static_cast<int*>(out)[i] = (int) q;
        } else if (is_byte_format(fmt)) {
            static_cast<unsigned char*>(out)[i] = byte_encode(fmt, (int) q);
        } else {
            unsigned char* p = static_cast<unsigned char*>(out) + 3 * (size_t) i;
            p[0] = (unsigned char) (q & 0xff);
            p[1] = (unsigned char) ((q >> 8) & 0xff);
            p[2] = (unsigned char) ((q >> 16) & 0xff);
        }
    }
    if (cfg->kind != R8BGPU_DITHER_OFF)
        for (int k = 0; k < kDitherTaps; k++) err_state[k] = eh[k];
    return 0;
}

int r8bgpu_batch_channel_groups(const r8bgpu_batch* b)
{
    if (b == nullptr) {
        set_err("batch_channel_groups: null batch");
        return -1;
    }
    if (b->mixed) { // parts run different plans: no two of their schedules are the same
        int n = 0;
        for (const auto& pb : b->mixed->parts) n += r8bgpu_batch_channel_groups(pb.get());
        return n;
    }
    // distinct schedules over every channel (of every shard)
    std::vector<const Schedule*> all;
    for (const r8bgpu_batch* sb : plan_batches(b)) {
        if (!sb->diverged) all.push_back(&sb->sched);
        else
            for (const Schedule& g : sb->rag.groups) all.push_back(&g);
    }
    int n = 0;
    for (size_t i = 0; i < all.size(); i++) {
        bool seen = false;
        for (size_t j = 0; j < i && !seen; j++) seen = same_state(*all[i], *all[j]);
        n += seen ? 0 : 1;
    }
    return n;
}

// ---- end of stream: flush channels (CDSPResampler::oneshot()'s tail, CDSPResampler.h:592-651) ------------------------
// Every named channel is fed silence until its output reaches its target (r8b_plan.h FlushPlan), returns the samples up
// to the target and is then cleared; the other channels take no input and keep their state.  The silence is never
// materialised: the first stage reads it through the records' `avail` (FlushView).

struct FlushJob {
    std::vector<int> named;                // the channels named, in the caller's order
    std::vector<int> key_of;               // per channel: index into plans (-1: not named; passthrough: 0, no plans)
    std::vector<FlushPlan> plans;          // per distinct (schedule group, target)
    std::vector<int> counts;               // per channel
    std::vector<long long> zero_from, out_base; // per channel: input and output totals before the flush
    int max_count = 0;
    size_t n_sub = 0;                      // sub-steps of the longest flush
};

// Validates a flush and plans it without changing any state.
static bool plan_batch_flush(r8bgpu_batch* b, const char* what, const int* channels, int n, const long long* targets,
                             bool have_out, int out_cap, FlushJob& job)
{
    const Plan& P = *b->plan;
    const std::string w(what);
    if (n < 0 || (n > 0 && channels == nullptr)) {
        set_err(w + ": bad arguments");
        return false;
    }
    if (n > 0 && has_fasttiming(P)) {
        set_err(w + ": R8B_FASTTIMING plans upload one position table per call and run lock-step only; they cannot "
                "flush channels on their own (feed silence with r8bgpu_batch_process)");
        return false;
    }
    if (n > 0 && targets == nullptr && P.trim_stage >= 0) {
        set_err(w + ": " + kTrimDefaultFlush);
        return false;
    }
    const size_t n_ch = (size_t) b->n_ch;
    job = FlushJob();
    job.key_of.assign(n_ch, -1);
    job.counts.assign(n_ch, 0);
    job.zero_from.assign(n_ch, 0);
    job.out_base.assign(n_ch, 0);
    const RaggedSchedule& rs = channel_schedules(b);
    std::map<std::pair<int, long long>, int> keys;
    return check_channels(b, channels, n, what, true, [&](int i, int c) {
        long long n_in = 0, n_out = 0;
        channel_totals_of(b, c, n_in, n_out);
        const long long T = targets != nullptr ? targets[i] : flush_default_target(P, n_in);
        if (T < 0) {
            set_err(w + (targets != nullptr ? ": negative target" : ": the default target does not fit a long long"));
            return false;
        }
        const long long cnt = std::max(0LL, T - n_out);
        if (cnt > out_cap || (cnt > 0 && !have_out)) {
            set_err(w + ": output capacity too small for this flush (channel " + std::to_string(c) + " returns " +
                    std::to_string(cnt) + " samples; r8bgpu_plan_flush_max_out_len() bounds a default flush)");
            return false;
        }
        job.counts[(size_t) c] = (int) cnt;
        job.max_count = std::max(job.max_count, (int) cnt);
        job.zero_from[(size_t) c] = n_in;
        job.out_base[(size_t) c] = n_out;
        job.named.push_back(c);
        if (P.passthrough) {
            job.key_of[(size_t) c] = 0;
            return true;
        }
        const int g = rs.group_of[(size_t) c];
        auto it = keys.find(std::make_pair(g, T));
        if (it == keys.end()) {
            it = keys.emplace(std::make_pair(g, T), (int) job.plans.size()).first;
            job.plans.emplace_back();
            plan_flush(rs.groups[(size_t) g], T, job.plans.back());
            job.n_sub = std::max(job.n_sub, job.plans.back().lens.size());
        }
        job.key_of[(size_t) c] = it->second;
        return true;
    });
}

// Queues the chain of every sub-step on st; channel c's output e lands at dst + c*stride + (e - out_base[c]).
static bool launch_flush(r8bgpu_batch* b, const FlushJob& job, double* dst, size_t stride, cudaStream_t st)
{
    const size_t n_ch = (size_t) b->n_ch;
    const FlushView fv{&job.zero_from, &job.out_base};
    for (size_t k = 0; k < job.n_sub; k++) {
        RaggedSchedule::Step step;
        step.key_of.assign(n_ch, 0);
        step.calls.emplace_back(b->plan->stages.size()); // key 0: channels without a part in this sub-step
        std::vector<int> key(job.plans.size(), -1);
        for (size_t c = 0; c < n_ch; c++) {
            const int p = job.key_of[c];
            if (p < 0 || k >= job.plans[(size_t) p].lens.size()) continue;
            if (key[(size_t) p] < 0) {
                key[(size_t) p] = (int) step.calls.size();
                step.calls.push_back(job.plans[(size_t) p].calls[k]);
            }
            step.key_of[c] = key[(size_t) p];
        }
        if (!launch_ragged(b, b->rag, step, nullptr, 0, dst, stride, st, nullptr, &fv)) return false;
    }
    return true;
}

// fp64 block (and, for typed output, a block of any format at 8 bytes per sample) of at least `need` samples per channel
static bool ensure_flush_staging(r8bgpu_batch* b, int need, bool raw)
{
    const size_t n_ch = (size_t) b->n_ch;
    if (b->fl_cap < (size_t) need) {
        b->fl_cap = (size_t) next_pow2(std::max(need, 64));
        b->fl_raw.reset(); // (rather than hold a block too small until the next typed flush)
    }
    return b->fl_out.grow(b->dev_bytes, b->fl_cap * n_ch, "flush: cudaMalloc(out)") &&
           (!raw || b->fl_raw.grow(b->dev_bytes, b->fl_cap * n_ch * 8, "flush: cudaMalloc(raw out)"));
}

// Each channel's count as the extent record of a ragged conversion (e1 - e0); returns the device records.
static const RaggedRec* upload_extents(r8bgpu_batch* b, const std::vector<int>& counts, cudaStream_t st)
{
    if (!ensure_ragged_state(b)) return nullptr;
    RaggedRec* h = b->rec.next("flush: records");
    if (h == nullptr) return nullptr;
    for (size_t c = 0; c < counts.size(); c++) {
        memset(&h[c], 0, sizeof h[c]);
        h[c].e1 = counts[c];
    }
    return b->rec.upload(0, counts.size(), st, "flush: record upload") ? (const RaggedRec*) b->rec.d : nullptr;
}

// Passthrough plans: the tail is counts[c] zeros, stored as silence_byte(format) in every byte of it -- zero bytes in
// the wide formats, the one byte that encodes 0 in U8, µ-law and A-law.  One 2-D fill per run of consecutive channels with
// equal counts (planar: rows, interleaved: columns).
static bool zero_fill(const r8bgpu_buffer& out, const std::vector<int>& counts, bool host, cudaStream_t st)
{
    const size_t e = (size_t) format_elem(out.format).bytes, n_ch = counts.size(); // outputs: one sample per element
    const int z = silence_byte(out.format);
    for (size_t c0 = 0; c0 < n_ch;) {
        size_t c1 = c0 + 1;
        while (c1 < n_ch && counts[c1] == counts[c0]) c1++;
        const size_t k = (size_t) counts[c0], nr = c1 - c0;
        unsigned char* p = (unsigned char*) out.data + (out.interleaved ? c0 * e : c0 * out.stride * e);
        const size_t width = (out.interleaved ? nr : k) * e, height = out.interleaved ? k : nr;
        if (k > 0) {
            if (host) {
                for (size_t r = 0; r < height; r++) memset(p + r * out.stride * e, z, width);
            } else if (!cuda_ok(cudaMemset2DAsync(p, out.stride * e, z, width, height, st), "flush: zero fill")) {
                return false;
            }
        }
        c0 = c1;
    }
    return true;
}

// The named channels return to the state after clear(): their rings are zeroed (one fill per ring and run of
// consecutive channels, in stream order after the flush's kernels) and their schedules restart.
static bool finish_flush(r8bgpu_batch* b, const FlushJob& job, cudaStream_t st)
{
    std::vector<int> ch = job.named;
    std::sort(ch.begin(), ch.end());
    for (const StageDev& d : b->dev) {
        if (d.ring == nullptr) continue;
        for (size_t i = 0; i < ch.size();) {
            size_t j = i + 1;
            while (j < ch.size() && ch[j] == ch[j - 1] + 1) j++;
            if (!cuda_ok(cudaMemsetAsync(d.ring + (size_t) ch[i] * (size_t) d.ring_cap, 0,
                                         (j - i) * (size_t) d.ring_cap * sizeof(double), st), "flush: cudaMemsetAsync"))
                return false;
            i = j;
        }
    }
    if (!dither_clear(b, ch.data(), (int) ch.size(), st)) return false;
    for (int c : ch) b->pass_n[(size_t) c] = 0;
    channel_schedules(b);
    b->rag.clear_channels(ch.data(), (int) ch.size());
    b->diverged = !b->rag.converged();
    if (!b->diverged) b->sched = b->rag.groups[0];
    return true;
}

// A chain whose last stage is a half-band upsampler writes outputs in pairs, so a flush cut at an odd target writes one
// spare sample past the channel's count (plan_flush): it must land in the batch's flush block, never in a caller's buffer.
static bool writes_pairs(const r8bgpu_batch* b)
{
    return !b->plan->stages.empty() && b->plan->stages.back().kind == ST_HBUP;
}

// Queues a planned flush on st into the device buffer `out` (host: into the batch's flush block fl_out, or a block that
// the conversion fills from it), then clears the named channels.  The chain writes straight into `out` only when `out`
// is plain fp64 and the chain writes nothing past a channel's count (or `out` is fl_out, whose rows keep one spare
// sample); otherwise it writes into fl_out and one ragged conversion copies exactly counts[c] samples of each channel
// into `out`.
static bool run_flush(r8bgpu_batch* b, const FlushJob& job, const r8bgpu_buffer& out, cudaStream_t st)
{
    const bool dith = job.max_count > 0 && dither_active(b, out.format, 0, b->n_ch);
    if (job.max_count > 0) {
        if (b->plan->passthrough) {
            if (!zero_fill(out, job.counts, false, st)) return false;
            if (dith) { // the dithered channels quantise their tail of zeros from an fp64 block of zeros
                if (!ensure_flush_staging(b, job.max_count, false)) return false;
                if (!cuda_ok(cudaMemsetAsync(b->fl_out, 0, b->fl_cap * (size_t) b->n_ch * sizeof(double), st), "flush: zero fill"))
                    return false;
            }
        } else if (buffer_is_plain(out) && (!writes_pairs(b) || out.data == b->fl_out)) {
            if (!launch_flush(b, job, (double*) out.data, out.stride, st)) return false;
        } else {
            if (!ensure_flush_staging(b, job.max_count + 1, false)) return false;
            if (!launch_flush(b, job, b->fl_out, b->fl_cap, st)) return false;
            const RaggedRec* rr = upload_extents(b, job.counts, st);
            if (rr == nullptr) return false;
            launch_from_f64(out.format, out.data, out.interleaved != 0, out.stride, b->fl_out, b->fl_cap, job.max_count, b->n_ch,
                            out.scale, st, rr);
            b->launches++;
        }
    }
    if (dith) {
        DitherRec* h = dither_records(b);
        if (h == nullptr) return false;
        for (int c = 0; c < b->n_ch; c++)
            h[c] = DitherRec{b->fl_out + (size_t) c * b->fl_cap, job.counts[(size_t) c], job.out_base[(size_t) c]};
        if (!dither_launch(b, out, 0, b->n_ch, st)) return false;
    }
    return finish_flush(b, job, st);
}

static int flush_host_impl(r8bgpu_batch* b, const int* channels, int n, const long long* targets, const r8bgpu_buffer& out,
                           int out_cap, int* counts)
{
    if (b->front) {
        const ShardFront& F = *b->front;
        if (n < 0 || (n > 0 && channels == nullptr)) {
            set_err("batch_flush_host: bad arguments");
            return -1;
        }
        if (!check_channels(b, channels, n, "batch_flush_host", true)) return -1;
        const std::vector<ChannelGroup> groups = group_channels(b, channels, n);
        std::vector<std::vector<long long>> tg(groups.size());
        if (targets != nullptr)
            for (size_t s = 0; s < groups.size(); s++) tg[s] = gather(targets, groups[s].idx);
        auto shard_targets = [&](int s) { return targets != nullptr ? tg[(size_t) s].data() : nullptr; };
        return front_call(
            b,
            [&](r8bgpu_batch* sb, int s) {
                const ChannelGroup& G = groups[(size_t) s];
                FlushJob dry;
                return plan_batch_flush(sb, "batch_flush_host", G.rows.data(), (int) G.rows.size(), shard_targets(s),
                                        out.data != nullptr, out_cap, dry);
            },
            [&](r8bgpu_batch* sb, int s) {
                const ChannelGroup& G = groups[(size_t) s];
                return flush_host_impl(sb, G.rows.data(), (int) G.rows.size(), shard_targets(s),
                                       shard_view(out, F.ch0[(size_t) s]), out_cap, counts + F.ch0[(size_t) s]);
            });
    }
    DeviceGuard g(b->device);
    FlushJob job;
    if (!plan_batch_flush(b, "batch_flush_host", channels, n, targets, out.data != nullptr, out_cap, job)) return -1;
    const int n_ch = b->n_ch;
    const cudaStream_t st = b->stream;
    bool ok = true;
    if (b->plan->passthrough && !dither_active(b, out.format, 0, n_ch)) {
        ok = zero_fill(out, job.counts, true, st) && finish_flush(b, job, st);
    } else if (job.max_count > 0) {
        const bool plain = buffer_is_plain(out);
        ok = ensure_flush_staging(b, job.max_count + 1, !plain); // the size run_flush asks for: no reallocation there
        const size_t cap = b->fl_cap;
        const r8bgpu_buffer dv = plain ? plain_buffer(b->fl_out, cap)
                                       : r8bgpu_buffer{b->fl_raw, out.format, out.interleaved, out.interleaved ? (size_t) n_ch : cap,
                                                       out.scale};
        ok = ok && run_flush(b, job, dv, st) && d2h_runs(out, dv, job.counts, st, "batch_flush_host");
    } else {
        ok = finish_flush(b, job, st);
    }
    ok = cuda_ok(cudaStreamSynchronize(st), "batch_flush_host: sync") && ok;
    if (!ok || !cuda_ok(cudaGetLastError(), "batch_flush_host: kernel launch")) return -1;
    for (int c = 0; c < n_ch; c++) counts[c] = job.counts[(size_t) c];
    return 0;
}

// ---- mixed batches: channel c runs plan plan_of[c] (r8bgpu_batch_create_mixed) ------------------------------------
// A call is planned on every part before any part runs, so a refused call changes no part.  Then, all on the batch
// stream st unless said otherwise: the call's records go up in one copy, one mapped conversion moves every channel's
// input from the caller's buffer into its row of its part's fp64 staging block, an event forks the parts onto their own
// streams where each runs its ragged chain, the batch stream waits for every part, and one mapped conversion moves every
// channel's output from its part's rows into the caller's buffer.  The host forms run the same sequence between the
// batch's raw blocks and synchronise.

// The host buffer for this call's records (its previous upload has finished).
static MapRec* mixed_records(r8bgpu_batch* b)
{
    return b->mixed->map.next("mixed: records");
}

static bool mixed_upload(r8bgpu_batch* b, size_t n, cudaStream_t st)
{
    return b->mixed->map.upload(0, n, st, "mixed: record upload");
}

// Every part's stream waits for what st has queued (the front conversion).
static void mixed_fork(r8bgpu_batch* b, cudaStream_t st)
{
    MixedFront& M = *b->mixed;
    cudaEventRecord(M.fork, st);
    for (const auto& pb : M.parts) cudaStreamWaitEvent(pb->stream, M.fork, 0);
}

// st waits for what every part's stream has queued (its chain).
static void mixed_join(r8bgpu_batch* b, cudaStream_t st)
{
    MixedFront& M = *b->mixed;
    for (size_t p = 0; p < M.parts.size(); p++) {
        cudaEventRecord(M.done[p], M.parts[p]->stream);
        cudaStreamWaitEvent(st, M.done[p], 0);
    }
}

// Host forms, in: the caller's samples cross PCIe as they are into the batch's raw block (h2d_ragged).  dv: the device
// view of that block.
static bool mixed_h2d(r8bgpu_batch* b, const r8bgpu_buffer& in, const int* lens, cudaStream_t st, r8bgpu_buffer& dv)
{
    MixedFront& M = *b->mixed;
    const size_t n_ch = (size_t) b->n_ch, in_cap = (size_t) b->plan->max_in_len;
    int max_len = 0;
    for (size_t c = 0; c < n_ch; c++) max_len = std::max(max_len, lens[c]);
    dv = r8bgpu_buffer{nullptr, in.format, in.interleaved, in.interleaved ? n_ch : in_cap, in.scale};
    if (max_len == 0) return true;
    if (!M.raw_in.grow(b->dev_bytes, n_ch * in_cap * 8, "mixed: cudaMalloc(raw in)")) return false;
    dv.data = M.raw_in;
    return h2d_ragged(in, lens, b->n_ch, M.raw_in, in_cap, st, "mixed");
}

// Host forms, out: the device view of the batch's raw output block for counts up to max_cnt.
static bool mixed_out_view(r8bgpu_batch* b, const r8bgpu_buffer& out, int max_cnt, r8bgpu_buffer& dv)
{
    MixedFront& M = *b->mixed;
    const size_t n_ch = (size_t) b->n_ch, w = staging_out_cap(std::max(max_cnt, 1));
    if (!M.raw_out.grow(b->dev_bytes, n_ch * w * 8, "mixed: cudaMalloc(raw out)")) return false;
    dv = r8bgpu_buffer{M.raw_out, out.format, out.interleaved, out.interleaved ? n_ch : w, out.scale};
    return true;
}

static int mixed_ragged(r8bgpu_batch* b, const char* what, const r8bgpu_buffer& in, const int* lens, const r8bgpu_buffer& out,
                        int out_cap, int* counts, bool host)
{
    MixedFront& M = *b->mixed;
    const std::string w(what);
    const int n_ch = b->n_ch;
    if (lens == nullptr) {
        set_err(w + ": null lens");
        return -1;
    }
    for (int c = 0; c < n_ch; c++)
        if (lens[c] < 0 || lens[c] > b->plan->max_in_len) {
            set_err(w + ": lens[" + std::to_string(c) + "] outside [0, MaxInLen]");
            return -1;
        }
    if (out_cap < M.max_out) {
        set_err(w + ": out_cap " + std::to_string(out_cap) + " is below r8bgpu_batch_max_out_len() = " + std::to_string(M.max_out));
        return -1;
    }
    DeviceGuard g(b->device);
    const size_t np = M.parts.size();
    std::vector<RaggedSchedule::Step> steps(np);
    std::vector<int> pl;
    for (size_t p = 0; p < np; p++) {
        pl.clear();
        for (int c : M.chans[p]) pl.push_back(lens[c]);
        r8bgpu_batch* pb = M.parts[p].get();
        if (!plan_ragged(pb, what, pl.data(), in.data != nullptr, out.data != nullptr, pb->plan->max_out_len, false, steps[p]))
            return -1;
    }
    // every part accepted the call
    for (const auto& pb : M.parts)
        if (!ensure_staging(pb.get())) return -1;
    const cudaStream_t st = b->stream;
    std::vector<int> cnt((size_t) n_ch);
    const bool dith = dither_active(b, out.format, 0, n_ch);
    const std::vector<long long> n0 = dith ? outputs_before(b) : std::vector<long long>();
    MapRec* h = mixed_records(b);
    if (h == nullptr) return -1;
    int max_len = 0, max_cnt = 0;
    for (int c = 0; c < n_ch; c++) {
        const size_t p = (size_t) M.part_of[(size_t) c], r = (size_t) M.row_of[(size_t) c];
        const r8bgpu_batch* pb = M.parts[p].get();
        const RaggedSchedule::Step& s = steps[p];
        const size_t o_cap = staging_out_cap(pb->plan->max_out_len);
        cnt[(size_t) c] = s.count[(size_t) s.key_of[r]];
        h[c] = MapRec{pb->st_in + r * (size_t) pb->plan->max_in_len, lens[c]};
        // a passthrough part hands its input back: the output row is the input row
        h[n_ch + c] = MapRec{pb->plan->passthrough ? h[c].row : pb->st_out + r * o_cap, cnt[(size_t) c]};
        max_len = std::max(max_len, lens[c]);
        max_cnt = std::max(max_cnt, cnt[(size_t) c]);
    }
    r8bgpu_buffer din = in, dout = out;
    bool ok = true;
    if (host) ok = mixed_h2d(b, in, lens, st, din) && mixed_out_view(b, out, max_cnt, dout);
    ok = ok && mixed_upload(b, 2 * (size_t) n_ch, st);
    if (ok) {
        launch_to_f64_mapped(din.format, din.data, din.interleaved != 0, din.stride, M.map.d, max_len, n_ch, din.scale, st);
        if (max_len > 0) b->launches++;
        mixed_fork(b, st);
        for (size_t p = 0; ok && p < np; p++) {
            r8bgpu_batch* pb = M.parts[p].get();
            if (!pb->plan->passthrough)
                ok = launch_ragged(pb, pb->rag, steps[p], pb->st_in, (size_t) pb->plan->max_in_len, pb->st_out,
                                   staging_out_cap(pb->plan->max_out_len), pb->stream);
        }
        mixed_join(b, st);
        launch_from_f64_mapped(dout.format, dout.data, dout.interleaved != 0, dout.stride, M.map.d + n_ch, max_cnt, n_ch,
                               dout.scale, st);
        if (max_cnt > 0) b->launches++;
        if (ok && dith) {
            DitherRec* dh = dither_records(b);
            ok = dh != nullptr;
            for (int c = 0; ok && c < n_ch; c++) dh[c] = DitherRec{h[n_ch + c].row, cnt[(size_t) c], n0[(size_t) c]};
            ok = ok && dither_launch(b, dout, 0, n_ch, st);
        }
    }
    if (host) {
        ok = ok && d2h_runs(out, dout, cnt, st, "mixed");
        ok = cuda_ok(cudaStreamSynchronize(st), (w + ": sync").c_str()) && ok;
    }
    if (!ok || !cuda_ok(cudaGetLastError(), (w + ": kernel launch").c_str())) return -1;
    for (int c = 0; c < n_ch; c++) counts[c] = cnt[(size_t) c];
    for (size_t p = 0; p < np; p++) adopt_step(M.parts[p].get(), steps[p]);
    return 0;
}

static int mixed_flush(r8bgpu_batch* b, const char* what, const int* channels, int n, const long long* targets,
                       const r8bgpu_buffer& out, int out_cap, int* counts, bool host)
{
    MixedFront& M = *b->mixed;
    const std::string w(what);
    const int n_ch = b->n_ch;
    if (n < 0 || (n > 0 && channels == nullptr)) {
        set_err(w + ": bad arguments");
        return -1;
    }
    if (!check_channels(b, channels, n, what, true)) return -1;
    const size_t np = M.parts.size();
    DeviceGuard g(b->device);
    std::vector<FlushJob> jobs(np);
    const std::vector<ChannelGroup> groups = group_channels(b, channels, n);
    for (size_t p = 0; p < np; p++) {
        const ChannelGroup& G = groups[p];
        const std::vector<long long> tg = targets != nullptr ? gather(targets, G.idx) : std::vector<long long>();
        if (!plan_batch_flush(G.b, what, G.rows.data(), (int) G.rows.size(), targets != nullptr ? tg.data() : nullptr,
                              out.data != nullptr, out_cap, jobs[p]))
            return -1;
    }
    // every part accepted the call
    for (size_t p = 0; p < np; p++)
        if (!M.parts[p]->plan->passthrough && jobs[p].max_count > 0 && !ensure_flush_staging(M.parts[p].get(), jobs[p].max_count + 1, false))
            return -1;
    const cudaStream_t st = b->stream;
    std::vector<int> cnt((size_t) n_ch), pass((size_t) n_ch, 0);
    MapRec* h = mixed_records(b);
    if (h == nullptr) return -1;
    int max_cnt = 0, max_all = 0;
    for (int c = 0; c < n_ch; c++) {
        const size_t p = (size_t) M.part_of[(size_t) c], r = (size_t) M.row_of[(size_t) c];
        const r8bgpu_batch* pb = M.parts[p].get();
        cnt[(size_t) c] = jobs[p].counts[r];
        max_all = std::max(max_all, cnt[(size_t) c]);
        if (pb->plan->passthrough) { // its tail is zeros, filled straight into the output
            pass[(size_t) c] = cnt[(size_t) c];
            h[c] = MapRec{nullptr, 0};
        } else {
            h[c] = MapRec{pb->fl_out + r * pb->fl_cap, cnt[(size_t) c]};
            max_cnt = std::max(max_cnt, cnt[(size_t) c]);
        }
    }
    r8bgpu_buffer dout = out;
    bool ok = !host || mixed_out_view(b, out, max_all, dout);
    ok = ok && mixed_upload(b, (size_t) n_ch, st);
    if (ok) {
        mixed_fork(b, st);
        for (size_t p = 0; ok && p < np; p++) {
            r8bgpu_batch* pb = M.parts[p].get();
            const FlushJob& job = jobs[p];
            if (job.named.empty()) continue;
            if (!pb->plan->passthrough && job.max_count > 0) ok = launch_flush(pb, job, pb->fl_out, pb->fl_cap, pb->stream);
            ok = ok && finish_flush(pb, job, pb->stream);
        }
        mixed_join(b, st);
        ok = ok && zero_fill(dout, pass, false, st);
        launch_from_f64_mapped(dout.format, dout.data, dout.interleaved != 0, dout.stride, M.map.d, max_cnt, n_ch, dout.scale, st);
        if (max_cnt > 0) b->launches++;
        if (ok && dither_active(b, out.format, 0, n_ch)) {
            // passthrough parts have no fp64 rows: their tails are read from a block of zeros, as in an ordinary batch
            DitherState& D = *b->dith;
            if (D.d_zero.size() < (size_t) max_all) {
                ok = D.d_zero.alloc(b->dev_bytes, (size_t) max_all, "flush: cudaMalloc(zeros)") &&
                     cuda_ok(cudaMemsetAsync(D.d_zero, 0, (size_t) max_all * sizeof(double), st), "flush: zero fill");
                if (!ok) D.d_zero.reset();
            }
            DitherRec* dh = ok ? dither_records(b) : nullptr;
            ok = ok && dh != nullptr;
            for (int c = 0; ok && c < n_ch; c++) {
                const Slot s = slot_of(b, c);
                dh[c] = DitherRec{h[c].row != nullptr ? h[c].row : D.d_zero, cnt[(size_t) c],
                                  jobs[(size_t) s.sub].out_base[(size_t) s.row], 0};
            }
            ok = ok && dither_launch(b, dout, 0, n_ch, st);
        }
        ok = ok && dither_clear(b, channels, n, st); // the flushed channels restart
    }
    if (host) {
        ok = ok && d2h_runs(out, dout, cnt, st, "mixed");
        ok = cuda_ok(cudaStreamSynchronize(st), (w + ": sync").c_str()) && ok;
    }
    if (!ok || !cuda_ok(cudaGetLastError(), (w + ": kernel launch").c_str())) return -1;
    for (int c = 0; c < n_ch; c++) counts[c] = cnt[(size_t) c];
    return 0;
}

r8bgpu_batch* r8bgpu_batch_create_mixed(const r8bgpu_plan* const* plans, int n_plans, const int* plan_of, int n_channels,
                                        int device)
{
    if (plans == nullptr || plan_of == nullptr || n_plans <= 0 || n_channels <= 0 || n_channels > 65535) {
        set_err("batch_create_mixed: need plans, plan_of and 1..65535 channels");
        return nullptr;
    }
    if (device == R8BGPU_DEVICE_ALL) {
        set_err("batch_create_mixed: a mixed batch runs on one device (R8BGPU_DEVICE_ALL is not supported; create one mixed "
                "batch per device)");
        return nullptr;
    }
    for (int p = 0; p < n_plans; p++) {
        if (plans[p] == nullptr) {
            set_err("batch_create_mixed: plans[" + std::to_string(p) + "] is null");
            return nullptr;
        }
        if (plans[p]->p.max_in_len != plans[0]->p.max_in_len) {
            set_err("batch_create_mixed: every plan must have the same MaxInLen (plans[" + std::to_string(p) + "] has " +
                    std::to_string(plans[p]->p.max_in_len) + ", plans[0] " + std::to_string(plans[0]->p.max_in_len) + ")");
            return nullptr;
        }
        if (has_fasttiming(plans[p]->p)) {
            set_err("batch_create_mixed: plans[" + std::to_string(p) + "] is an R8B_FASTTIMING plan, which runs lock-step only");
            return nullptr;
        }
    }
    std::vector<std::vector<int>> chans((size_t) n_plans);
    for (int c = 0; c < n_channels; c++) {
        if (plan_of[c] < 0 || plan_of[c] >= n_plans) {
            set_err("batch_create_mixed: plan_of[" + std::to_string(c) + "] is not a plan index");
            return nullptr;
        }
        chans[(size_t) plan_of[c]].push_back(c);
    }
    for (int p = 0; p < n_plans; p++)
        if (chans[(size_t) p].empty()) {
            set_err("batch_create_mixed: plans[" + std::to_string(p) + "] has no channel");
            return nullptr;
        }
    int ndev = 0;
    if (!cuda_ok(cudaGetDeviceCount(&ndev), "batch_create_mixed: cudaGetDeviceCount") || ndev == 0) {
        if (g_err.empty() || ndev == 0) set_err("batch_create_mixed: no CUDA device (this engine has no CPU fallback)");
        return nullptr;
    }
    if (device < 0 && !cuda_ok(cudaGetDevice(&device), "batch_create_mixed: cudaGetDevice")) return nullptr;
    if (device >= ndev) {
        set_err("batch_create_mixed: device index out of range");
        return nullptr;
    }
    DeviceGuard g(device);
    if (!g.ok) {
        set_err("batch_create_mixed: cudaSetDevice failed");
        return nullptr;
    }
    std::unique_ptr<r8bgpu_batch> b(new r8bgpu_batch);
    b->plan_copy = plans[0]->p; // (its MaxInLen is every plan's; nothing else of it is used)
    b->plan = &b->plan_copy;
    b->n_ch = n_channels;
    b->device = device;
    b->mixed.reset(new MixedFront);
    MixedFront& M = *b->mixed;
    M.part_of.assign((size_t) n_channels, 0);
    M.row_of.assign((size_t) n_channels, 0);
    M.chans = chans;
    for (int p = 0; p < n_plans; p++) {
        for (size_t r = 0; r < chans[(size_t) p].size(); r++) {
            M.part_of[(size_t) chans[(size_t) p][r]] = p;
            M.row_of[(size_t) chans[(size_t) p][r]] = (int) r;
        }
        M.max_out = std::max(M.max_out, plans[p]->p.max_out_len);
        if (plans[p]->p.trim_stage < 0) // (trim parts take explicit flush targets only)
            M.flush_max_out = std::max(M.flush_max_out, flush_max_out_len(plans[p]->p));
        M.parts.emplace_back(r8bgpu_batch_create(plans[p], (int) chans[(size_t) p].size(), device));
        if (M.parts.back() == nullptr) return nullptr; // (b's destructor releases the parts made so far)
        M.streams.emplace_back();
        M.done.emplace_back();
        if (!cuda_ok(cudaStreamCreateWithFlags(M.streams.back().put(), cudaStreamNonBlocking), "batch_create_mixed: stream"))
            return nullptr;
        M.parts.back()->stream = M.streams.back(); // the part was created on the legacy stream and has finished its clear()
        if (!cuda_ok(cudaEventCreateWithFlags(M.done.back().put(), cudaEventDisableTiming), "batch_create_mixed: event"))
            return nullptr;
    }
    if (!cuda_ok(cudaEventCreateWithFlags(M.fork.put(), cudaEventDisableTiming), "batch_create_mixed: event") ||
        !M.map.create(b->dev_bytes, 2 * (size_t) n_channels, "batch_create_mixed: cudaMalloc(records)",
                      "batch_create_mixed: cudaMallocHost(records)", "batch_create_mixed: event"))
        return nullptr;
    return b.release();
}

int r8bgpu_batch_max_out_len(const r8bgpu_batch* b)
{
    if (b == nullptr) {
        set_err("batch_max_out_len: null batch");
        return -1;
    }
    const int n = b->mixed ? b->mixed->max_out : b->plan->max_out_len;
    return dsd_on(b) ? dsd_out_bound(n) : n;
}

int r8bgpu_batch_flush_max_out_len(const r8bgpu_batch* b)
{
    if (b == nullptr) {
        set_err("batch_flush_max_out_len: null batch");
        return -1;
    }
    if (!b->mixed && b->plan->trim_stage >= 0) {
        set_err(std::string("batch_flush_max_out_len: ") + kTrimDefaultFlush);
        return -1;
    }
    const int n = b->mixed ? b->mixed->flush_max_out : flush_max_out_len(*b->plan);
    return dsd_on(b) ? dsd_flush_bound(n) : n;
}

r8bgpu_batch* r8bgpu_batch_part(r8bgpu_batch* b, int plan_index)
{
    if (b == nullptr || !b->mixed || plan_index < 0 || plan_index >= (int) b->mixed->parts.size()) {
        set_err("batch_part: not a mixed batch, or plan index out of range");
        return nullptr;
    }
    return b->mixed->parts[(size_t) plan_index].get();
}

int r8bgpu_batch_flush(r8bgpu_batch* b, const int* channels, int n, const long long* targets, const r8bgpu_buffer* d_out,
                       int out_cap, int* counts)
{
    if (b == nullptr || counts == nullptr) {
        set_err("batch_flush: null batch or counts");
        return -1;
    }
    if (refuse_front_device(b, "batch_flush")) return -1;
    if (!check_buffer(b, d_out, "batch_flush(out)", true)) return -1;
    if (dsd_on(b)) return dsd_flush(b, "batch_flush", channels, n, targets, *d_out, out_cap, counts, false);
    if (b->mixed) return mixed_flush(b, "batch_flush", channels, n, targets, *d_out, out_cap, counts, false);
    DeviceGuard g(b->device);
    FlushJob job;
    if (!plan_batch_flush(b, "batch_flush", channels, n, targets, d_out->data != nullptr, out_cap, job)) return -1;
    if (!run_flush(b, job, *d_out, b->stream)) return -1;
    if (!cuda_ok(cudaGetLastError(), "batch_flush: kernel launch")) return -1;
    for (int c = 0; c < b->n_ch; c++) counts[c] = job.counts[(size_t) c];
    return 0;
}

int r8bgpu_batch_flush_host(r8bgpu_batch* b, const int* channels, int n, const long long* targets, const r8bgpu_buffer* h_out,
                            int out_cap, int* counts)
{
    if (b == nullptr || counts == nullptr) {
        set_err("batch_flush_host: null batch or counts");
        return -1;
    }
    if (!check_buffer(b, h_out, "batch_flush_host(out)", true)) return -1;
    if (dsd_on(b)) return dsd_flush(b, "batch_flush_host", channels, n, targets, *h_out, out_cap, counts, true);
    if (b->mixed) return mixed_flush(b, "batch_flush_host", channels, n, targets, *h_out, out_cap, counts, true);
    return flush_host_impl(b, channels, n, targets, *h_out, out_cap, counts);
}

int r8bgpu_batch_channel_totals(const r8bgpu_batch* b, long long* n_in, long long* n_out)
{
    if (b == nullptr || n_in == nullptr || n_out == nullptr) {
        set_err("batch_channel_totals: null argument");
        return -1;
    }
    for (int c = 0; c < b->n_ch; c++) channel_totals_of(b, c, n_in[c], n_out[c]);
    return 0;
}

int r8bgpu_batch_process_host(r8bgpu_batch* b, const double* h_in, size_t in_stride, int l, double* h_out,
                              size_t out_stride, int out_cap)
{
    if (b == nullptr) {
        set_err("batch_process_host: null batch");
        return -1;
    }
    if (refuse_dsd_plain(b, "batch_process_host")) return -1;
    const r8bgpu_buffer in = { const_cast<double*>(h_in), R8BGPU_F64, 0, in_stride, 1.0 };
    const r8bgpu_buffer out = { h_out, R8BGPU_F64, 0, out_stride, 1.0 };
    return process_host_impl(b, in, l, out, out_cap);
}

int r8bgpu_batch_process_host_fmt(r8bgpu_batch* b, const r8bgpu_buffer* h_in, int l, const r8bgpu_buffer* h_out,
                                  int out_cap)
{
    if (b == nullptr) {
        set_err("batch_process_host_fmt: null batch");
        return -1;
    }
    if (!check_buffer(b, h_in, "batch_process_host_fmt(in)") || !check_buffer(b, h_out, "batch_process_host_fmt(out)", true) ||
        !check_lengths(*h_in, &l, 1, "batch_process_host_fmt"))
        return -1;
    if (dsd_on(b)) {
        if (refuse_mixed_lockstep(b, "batch_process_host_fmt")) return -1;
        return dsd_process(b, "batch_process_host_fmt", *h_in, l, nullptr, *h_out, out_cap, nullptr, true);
    }
    return process_host_impl(b, *h_in, l, *h_out, out_cap);
}

// Device buffers in any format: widen into the staging block, run, narrow into the caller's buffer --
// all on the batch stream, asynchronous like r8bgpu_batch_process().
int r8bgpu_batch_process_fmt(r8bgpu_batch* b, const r8bgpu_buffer* d_in, int l, const r8bgpu_buffer* d_out,
                             int out_cap)
{
    if (b == nullptr) {
        set_err("batch_process_fmt: null batch");
        return -1;
    }
    if (refuse_mixed_lockstep(b, "batch_process_fmt")) return -1;
    if (refuse_front_device(b, "batch_process_fmt")) return -1;
    if (!check_buffer(b, d_in, "batch_process_fmt(in)") || !check_buffer(b, d_out, "batch_process_fmt(out)", true) ||
        !check_lengths(*d_in, &l, 1, "batch_process_fmt"))
        return -1;
    if (dsd_on(b)) return dsd_process(b, "batch_process_fmt", *d_in, l, nullptr, *d_out, out_cap, nullptr, false);
    if (buffer_is_plain(*d_in) && buffer_is_plain(*d_out))
        return r8bgpu_batch_process(b, (const double*) d_in->data, d_in->stride, l, (double*) d_out->data,
                                    d_out->stride, out_cap);
    return process_dev(b, "batch_process_fmt", *d_in, l, *d_out, out_cap);
}

// ---- one-bit DSD output (r8b_dsdmod.cuh; the walk, K8, in r8b_dsd_mod.cu) -------------------------------------------
// A call runs the resampler as for fp64 output into the batch's rows (DsdOutState::d_y), then k_dsd_mod turns each
// channel's rows into whole bytes after the bits it held back, and holds back the bits of an unfinished byte.  The bytes
// are therefore a function of the channel's fp64 stream alone.

static bool dsd_rate_ok(double r)
{
    for (double base : {44100.0, 48000.0})
        for (int m : {64, 128, 256, 512})
            if (r == base * m) return true;
    return false;
}

// The fp64 rows hold at least `need` samples per channel.
static bool dsd_rows(r8bgpu_batch* b, size_t need)
{
    DsdOutState& D = *b->dsd;
    if (D.y_cap >= need) return true;
    if (!D.d_y.grow(b->dev_bytes, need * (size_t) b->n_ch, "dsd: cudaMalloc(rows)")) return false;
    D.y_cap = need;
    return true;
}

static bool dsd_check_out(const r8bgpu_batch* b, const std::string& what, const r8bgpu_buffer& out)
{
    if (is_dsd_format(out.format)) return true;
    set_err(what + ": DSD output is on (r8bgpu_batch_set_dsd_out): the output must be R8BGPU_DSD_LSB or R8BGPU_DSD_MSB");
    return false;
}

// Checks a processing call against the DSD rules on b (ordinary or mixed) without changing anything.
static bool dsd_check_process(const r8bgpu_batch* b, const std::string& what, const r8bgpu_buffer& out, int out_cap, bool lockstep)
{
    if (!dsd_check_out(b, what, out)) return false;
    const int bound = dsd_out_bound(b->mixed ? b->mixed->max_out : b->plan->max_out_len);
    if (out_cap < bound) {
        set_err(what + ": out_cap " + std::to_string(out_cap) + " is below r8bgpu_batch_max_out_len() = " + std::to_string(bound) +
                " (DSD output is on)");
        return false;
    }
    if (!lockstep) return true;
    if (b->diverged) {
        set_err(what + ": " + kDivergedTyped);
        return false;
    }
    const std::vector<int>& p = b->dsd->pend;
    if (std::any_of(p.begin(), p.end(), [&](int k) { return k != p[0]; })) {
        set_err(what + ": the channels hold back different numbers of DSD bits (after ragged calls); use the ragged calls");
        return false;
    }
    return true;
}

// The call's block lengths L (a lock-step call's l for every channel) are in [0, MaxInLen] and have an input.
static bool dsd_check_lengths(const r8bgpu_batch* b, const std::string& what, const r8bgpu_buffer& in, const int* L, bool lockstep)
{
    for (int c = 0; c < b->n_ch; c++)
        if (L[c] < 0 || L[c] > b->plan->max_in_len) {
            set_err(what + (lockstep ? ": l must be in [0, MaxInLen]" : ": lens[" + std::to_string(c) + "] outside [0, MaxInLen]"));
            return false;
        }
    if (in.data == nullptr && std::any_of(L, L + b->n_ch, [](int k) { return k > 0; })) {
        set_err(what + ": null input");
        return false;
    }
    return true;
}

// Modulates the rows of this call: channel c's cnt[c] samples, then zeros[c] of silence (nullptr: none), after its
// held-back bits; the channels with clear[c] restart afterwards.  Writes the whole bytes into `out` (device), or through
// the batch's byte block into `out` (host; synchronises).  bits[c]: the bits written.
static bool dsd_modulate(r8bgpu_batch* b, const char* what, const std::vector<int>& cnt, const std::vector<int>* zeros,
                         const std::vector<char>* clear, const r8bgpu_buffer& out, bool host, std::vector<int>& bits)
{
    DsdOutState& D = *b->dsd;
    const int n_ch = b->n_ch;
    const cudaStream_t st = b->stream;
    DsdModRec* h = D.rec.next("dsd: records");
    if (h == nullptr) return false;
    bits.assign((size_t) n_ch, 0);
    std::vector<int> next((size_t) n_ch), nbytes((size_t) n_ch);
    bool work = false;
    int max_bytes = 0;
    for (int c = 0; c < n_ch; c++) {
        const size_t i = (size_t) c;
        const int z = zeros ? (*zeros)[i] : 0, clr = clear ? (*clear)[i] : 0;
        h[c] = DsdModRec{D.d_y + i * D.y_cap, cnt[i], z, D.pend[i], clr};
        const long long tot = (long long) D.pend[i] + cnt[i] + z;
        bits[i] = (int) (tot & ~7LL);
        nbytes[i] = bits[i] / 8;
        next[i] = clr ? 0 : (int) (tot & 7);
        max_bytes = std::max(max_bytes, nbytes[i]);
        work = work || tot > D.pend[i] || clr;
    }
    r8bgpu_buffer dv = out;
    if (host) {
        const size_t w = out.interleaved ? (size_t) n_ch : (size_t) std::max(max_bytes, 1);
        if (!D.d_bytes.grow(b->dev_bytes, w * (out.interleaved ? (size_t) std::max(max_bytes, 1) : (size_t) n_ch),
                            "dsd: cudaMalloc(bytes)"))
            return false;
        dv = r8bgpu_buffer{D.d_bytes, out.format, out.interleaved, w, out.scale};
    }
    bool ok = true;
    if (work) {
        ok = D.rec.upload(0, (size_t) n_ch, st, "dsd: record upload");
        // with timing on, K8 is timed as the stage after the plan's last (r8bgpu_batch_stage_time_ms)
        r8bgpu_batch::EvPair ev = ok ? time_begin(b, (int) b->plan->stages.size(), st) : r8bgpu_batch::EvPair{};
        ok = ok && cuda_ok(launch_dsd_mod(D.rec.d, D.d_state, dv.data, dv.interleaved != 0, dv.stride, out.format == FMT_DSD_MSB,
                                          out.scale, n_ch, st),
                           "dsd: k_dsd_mod launch");
        time_end(b, ev, st);
        b->launches++;
    }
    if (host) {
        ok = ok && d2h_runs(out, dv, nbytes, st, what);
        ok = cuda_ok(cudaStreamSynchronize(st), (std::string(what) + ": sync").c_str()) && ok;
    }
    if (!ok) return false;
    D.pend.swap(next);
    return true;
}

// A processing call with DSD output.  lens == nullptr: a lock-step call of l samples (returns the common count), else a
// ragged one (returns 0).  Host forms: the caller's input crosses PCIe as it is into a device block first, and the
// bytes come back once modulated.
static int dsd_process(r8bgpu_batch* b, const char* what, const r8bgpu_buffer& in, int l, const int* lens,
                       const r8bgpu_buffer& out, int out_cap, int* counts, bool host)
{
    const std::string w(what);
    const bool lockstep = lens == nullptr;
    if (b->front) { // (host forms only) each shard runs its channel range once every shard has accepted the call
        const ShardFront& F = *b->front;
        return front_call(
            b,
            [&](r8bgpu_batch* sb, int s) {
                if (!lockstep) { // everything the shard's run checks, and its ragged schedule, without running it
                    const int* L = lens + F.ch0[(size_t) s];
                    RaggedSchedule::Step dry;
                    return dsd_check_process(sb, w, out, out_cap, false) && dsd_check_lengths(sb, w, in, L, false) &&
                           plan_ragged(sb, what, L, in.data != nullptr, true, (int) staging_out_cap(sb->plan->max_out_len),
                                       false, dry);
                }
                const std::vector<int> lk((size_t) sb->n_ch, l);
                return dsd_check_process(sb, w, out, out_cap, true) && dsd_check_lengths(sb, w, in, lk.data(), true) &&
                       (sb->dsd->pend[0] == F.shards[0]->dsd->pend[0] ||
                        (set_err(w + ": the channels hold back different numbers of DSD bits (after ragged calls); use the "
                                     "ragged calls"),
                         false));
            },
            [&](r8bgpu_batch* sb, int s) {
                const int c0 = F.ch0[(size_t) s];
                return dsd_process(sb, what, shard_view(in, c0), l, lockstep ? nullptr : lens + c0, shard_view(out, c0), out_cap,
                                   counts != nullptr ? counts + c0 : nullptr, true);
            });
    }
    DsdOutState& D = *b->dsd;
    const int n_ch = b->n_ch;
    const size_t in_cap = (size_t) b->plan->max_in_len;
    const std::vector<int> lk(lockstep ? (size_t) n_ch : 0, l);
    const int* L = lockstep ? lk.data() : lens;
    if (!dsd_check_process(b, w, out, out_cap, lockstep) || !dsd_check_lengths(b, w, in, L, lockstep)) return -1;
    DeviceGuard g(b->device);
    if (!dsd_rows(b, staging_out_cap(b->mixed ? b->mixed->max_out : b->plan->max_out_len))) return -1;
    const cudaStream_t st = b->stream;
    r8bgpu_buffer din = in;
    if (host && b->mixed) {
        if (!mixed_h2d(b, in, L, st, din)) return -1;
    } else if (host) {
        if (!D.d_in.grow(b->dev_bytes, (size_t) n_ch * in_cap * 8, "dsd: cudaMalloc(in)")) return -1;
        din = r8bgpu_buffer{D.d_in, in.format, in.interleaved, in.interleaved ? (size_t) n_ch : in_cap, in.scale};
        if (!h2d_ragged(in, L, n_ch, D.d_in, in_cap, st, what)) return -1;
    }
    const r8bgpu_buffer y = plain_buffer(D.d_y, D.y_cap);
    std::vector<int> cnt((size_t) n_ch);
    if (lockstep) {
        const int n = process_dev(b, what, din, l, y, (int) D.y_cap);
        if (n < 0) return -1;
        std::fill(cnt.begin(), cnt.end(), n);
    } else if ((b->mixed ? mixed_ragged(b, what, din, lens, y, (int) D.y_cap, cnt.data(), false)
                         : process_ragged_dev(b, din, lens, y, (int) D.y_cap, cnt.data(), false)) < 0) {
        return -1;
    }
    std::vector<int> bits;
    if (!dsd_modulate(b, what, cnt, nullptr, nullptr, out, host, bits)) return -1;
    if (counts != nullptr)
        for (int c = 0; c < n_ch; c++) counts[c] = bits[(size_t) c];
    return lockstep ? bits[0] : 0;
}

// Checks a flush against the DSD rules on b (ordinary or mixed) without changing anything.
static bool dsd_check_flush(const r8bgpu_batch* b, const std::string& what, const int* channels, int n, const long long* targets,
                            const r8bgpu_buffer& out, int out_cap)
{
    if (!dsd_check_out(b, what, out)) return false;
    if (n < 0 || (n > 0 && channels == nullptr)) {
        set_err(what + ": bad arguments");
        return false;
    }
    return check_channels(b, channels, n, what.c_str(), true, [&](int i, int c) {
        if (targets != nullptr && targets[i] % 8 != 0) {
            set_err(what + ": flush targets must be multiples of 8 samples while DSD output is on (channel " + std::to_string(c) + ")");
            return false;
        }
        long long n_in = 0, n_out = 0;
        channel_totals_of(b, c, n_in, n_out);
        const Slot s = slot_of(b, c);
        const long long T = targets != nullptr ? targets[i] : flush_default_target(*s.b->plan, n_in);
        const long long bits = ((long long) b->dsd->pend[(size_t) c] + std::max(0LL, T - n_out) + 7) / 8 * 8;
        if (T >= 0 && bits > out_cap) {
            set_err(what + ": output capacity too small for this flush (channel " + std::to_string(c) + " returns " +
                    std::to_string(bits) + " DSD samples; r8bgpu_batch_flush_max_out_len() bounds a default flush)");
            return false;
        }
        return true;
    });
}

static int dsd_flush(r8bgpu_batch* b, const char* what, const int* channels, int n, const long long* targets,
                     const r8bgpu_buffer& out, int out_cap, int* counts, bool host)
{
    const std::string w(what);
    if (b->front) {
        const ShardFront& F = *b->front;
        if (n < 0 || (n > 0 && channels == nullptr)) {
            set_err(w + ": bad arguments");
            return -1;
        }
        if (!check_channels(b, channels, n, what, true)) return -1;
        const std::vector<ChannelGroup> groups = group_channels(b, channels, n);
        std::vector<std::vector<long long>> tg(groups.size());
        if (targets != nullptr)
            for (size_t s = 0; s < groups.size(); s++) tg[s] = gather(targets, groups[s].idx);
        auto shard_targets = [&](int s) { return targets != nullptr ? tg[(size_t) s].data() : nullptr; };
        return front_call(
            b,
            [&](r8bgpu_batch* sb, int s) {
                const ChannelGroup& G = groups[(size_t) s];
                FlushJob dry;
                return dsd_check_flush(sb, w, G.rows.data(), (int) G.rows.size(), shard_targets(s), out, out_cap) &&
                       plan_batch_flush(sb, what, G.rows.data(), (int) G.rows.size(), shard_targets(s), true, INT_MAX, dry);
            },
            [&](r8bgpu_batch* sb, int s) {
                const ChannelGroup& G = groups[(size_t) s];
                return dsd_flush(sb, what, G.rows.data(), (int) G.rows.size(), shard_targets(s), shard_view(out, F.ch0[(size_t) s]),
                                 out_cap, counts + F.ch0[(size_t) s], true);
            });
    }
    if (!dsd_check_flush(b, w, channels, n, targets, out, out_cap)) return -1;
    const int n_ch = b->n_ch;
    DeviceGuard g(b->device);
    std::vector<int> cnt((size_t) n_ch, 0);
    const cudaStream_t st = b->stream;
    if (b->mixed) {
        // (the parts' counts are known before anything runs; the rows are sized for the largest)
        int need = 0;
        for (int i = 0; i < n; i++) {
            long long n_in = 0, n_out = 0;
            channel_totals_of(b, channels[i], n_in, n_out);
            const Slot s = slot_of(b, channels[i]);
            const long long T = targets != nullptr ? targets[i] : flush_default_target(*s.b->plan, n_in);
            need = (int) std::max<long long>(need, std::min<long long>(INT_MAX - 8, std::max(0LL, T - n_out)));
        }
        if (!dsd_rows(b, staging_out_cap(std::max(need, 1))) ||
            mixed_flush(b, what, channels, n, targets, plain_buffer(b->dsd->d_y, b->dsd->y_cap), (int) b->dsd->y_cap, cnt.data(),
                        false) < 0)
            return -1;
    } else {
        FlushJob job;
        if (!plan_batch_flush(b, what, channels, n, targets, true, INT_MAX, job)) return -1;
        if (!dsd_rows(b, staging_out_cap(std::max(job.max_count, 1))) ||
            !run_flush(b, job, plain_buffer(b->dsd->d_y, b->dsd->y_cap), st) ||
            !cuda_ok(cudaGetLastError(), (w + ": kernel launch").c_str()))
            return -1;
        cnt = job.counts;
    }
    // every named channel ends on a whole byte and restarts
    std::vector<int> zeros((size_t) n_ch, 0);
    std::vector<char> clear((size_t) n_ch, 0);
    for (int i = 0; i < n; i++) {
        const size_t c = (size_t) channels[i];
        zeros[c] = (int) ((8 - (b->dsd->pend[c] + cnt[c]) % 8) % 8);
        clear[c] = 1;
    }
    std::vector<int> bits;
    if (!dsd_modulate(b, what, cnt, &zeros, &clear, out, host, bits)) return -1;
    for (int c = 0; c < n_ch; c++) counts[c] = bits[(size_t) c];
    return 0;
}

int r8bgpu_batch_set_dsd_out(r8bgpu_batch* b, int on)
{
    if (b == nullptr) {
        set_err("batch_set_dsd_out: null batch");
        return -1;
    }
    if (on) { // every plan must end at a DSD rate (refused before anything changes)
        for (const r8bgpu_batch* pb : plan_batches(b))
            if (!dsd_rate_ok(pb->plan->dst_rate)) {
                char msg[200];
                snprintf(msg, sizeof msg, "batch_set_dsd_out: destination rate %.17g is not a DSD rate (64, 128, 256 or 512 x "
                         "44100 or 48000)", pb->plan->dst_rate);
                set_err(msg);
                return -1;
            }
    }
    if (b->front) {
        for (const auto& sb : b->front->shards)
            if (r8bgpu_batch_set_dsd_out(sb.get(), on) != 0) return -1;
        return 0;
    }
    DeviceGuard g(b->device);
    // queued calls use the state they were queued with
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "batch_set_dsd_out: sync")) return -1;
    if (!on) {
        b->dsd.reset();
        return 0;
    }
    const size_t n_ch = (size_t) b->n_ch;
    if (!b->dsd) {
        std::unique_ptr<DsdOutState> D(new DsdOutState);
        D->pend.assign(n_ch, 0);
        if (!D->d_state.alloc(b->dev_bytes, n_ch, "batch_set_dsd_out: cudaMalloc") ||
            !D->rec.create(b->dev_bytes, n_ch, "batch_set_dsd_out: cudaMalloc", "batch_set_dsd_out: cudaMallocHost",
                           "batch_set_dsd_out: cudaEventCreate"))
            return -1;
        b->dsd = std::move(D);
    }
    // turning it on (again) starts every channel's modulator afresh
    return dsd_clear(b, nullptr, 0, b->stream) && cuda_ok(cudaStreamSynchronize(b->stream), "batch_set_dsd_out: sync") ? 0 : -1;
}

int r8bgpu_batch_dsd_overloads(r8bgpu_batch* b, long long* counts)
{
    if (b == nullptr || counts == nullptr) {
        set_err("batch_dsd_overloads: null argument");
        return -1;
    }
    if (!dsd_on(b)) {
        set_err("batch_dsd_overloads: DSD output is off (r8bgpu_batch_set_dsd_out)");
        return -1;
    }
    if (b->front) {
        for (size_t s = 0; s < b->front->shards.size(); s++)
            if (r8bgpu_batch_dsd_overloads(b->front->shards[s].get(), counts + b->front->ch0[s]) != 0) return -1;
        return 0;
    }
    DeviceGuard g(b->device);
    std::vector<DsdModState> h((size_t) b->n_ch);
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "batch_dsd_overloads: sync") ||
        !cuda_ok(cudaMemcpy(h.data(), b->dsd->d_state, h.size() * sizeof(DsdModState), cudaMemcpyDeviceToHost),
                 "batch_dsd_overloads: copy"))
        return -1;
    for (int c = 0; c < b->n_ch; c++) counts[c] = h[(size_t) c].overloads;
    return 0;
}

int r8bgpu_dsd_modulate_host(double scale, const double* y, int n, double* state, unsigned char* bits, long long* overloads)
{
    if (n < 0 || (n > 0 && (y == nullptr || bits == nullptr)) || state == nullptr || overloads == nullptr) {
        set_err("dsd_modulate_host: bad arguments");
        return -1;
    }
    DsdFilter f;
    f.ep = state[0];
    for (int k = 0; k < 7; k++) f.p[k] = state[k + 1];
    long long ov = 0;
    for (int i = 0; i < n; i++) bits[i] = (unsigned char) dsd_mod_step(f, dsd_mod_input(y[i], scale), ov);
    state[0] = f.ep;
    for (int k = 0; k < 7; k++) state[k + 1] = f.p[k];
    *overloads += ov;
    return 0;
}

double r8bgpu_measure_fp64_tflops(int device)
{
    int dev = device;
    if (dev < 0 && !cuda_ok(cudaGetDevice(&dev), "measure_fp64")) return -1.0;
    DeviceGuard guard(dev);
    if (!guard.ok) {
        set_err("measure_fp64: cannot select device");
        return -1.0;
    }
    const double tf = measure_dfma_tflops();
    if (tf < 0.0) cuda_ok(cudaGetLastError(), "measure_fp64");
    return tf;
}

void* r8bgpu_host_alloc(size_t bytes)
{
    void* p = nullptr;
    if (!cuda_ok(cudaMallocHost(&p, bytes), "host_alloc")) return nullptr;
    return p;
}

void r8bgpu_host_free(void* p)
{
    if (p == nullptr) return;
    if (!numa_host_free(p)) cudaFreeHost(p);
}

} // extern "C"

// ---- moving streams: a channel's complete state as a blob (include/r8bgpu.h, r8b_state.cu) ---------------------------
// A blob is what a fresh slot needs to continue the stream bit for bit: the schedule of its group, pass_n, the trim factor,
// the dither setting and history, and for every stage input j the window [n_in_j - H_j, n_in_j) of that stream.  Kernels
// are pure functions of (ring windows, schedule) addressed by absolute sample index, so these pieces are the whole stream.

namespace {

constexpr uint32_t kStateMagic = 0x53423852u; // "R8BS", little-endian
constexpr uint32_t kStateVersion = 1;

// The blob's first 32 words.  Fields are little-endian; words 3..10 are the plan's fingerprint.
struct StateHeader {
    uint32_t magic, version;
    uint64_t sum;   // checksum of every other word of the blob (state_word_term)
    uint64_t bytes; // the blob's length
    double src, dst;
    int32_t max_in_len, extfft;
    double trans_band, atten;
    int32_t fasttiming, n_stages;
    double max_trim;
    uint64_t design; // hash of the designed stage data (design_hash)
    int64_t pass_n;
    double trim;
    int32_t dither_kind, dither_taps;
    uint64_t dither_seed;
    double taps[16];
    int64_t m; // dithered outputs since the stream's clear
};
// Then one record per stage, the 16-slot dither error history, and the windows in stage order.
struct StateStage {
    int64_t n_in, n_out;
    int32_t in_counter, in_pos_int;
    double in_pos_shift, fpos;
    int64_t p;
    double dsr;
    int64_t window; // H_j
};
static_assert(sizeof(StateHeader) == 32 * 8 && sizeof(StateStage) == 8 * 8, "blob layout");
constexpr size_t kFpFirst = offsetof(StateHeader, src), kFpEnd = offsetof(StateHeader, pass_n);

unsigned long long fnv(unsigned long long h, const void* p, size_t n)
{
    const unsigned char* c = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < n; i++) h = (h ^ c[i]) * 1099511628211ull;
    return h;
}
template <class T> unsigned long long fnv_v(unsigned long long h, const std::vector<T>& v)
{
    const unsigned long long n = v.size();
    h = fnv(h, &n, sizeof n);
    return v.empty() ? h : fnv(h, v.data(), v.size() * sizeof(T));
}

// Every number the planner designed: stage kinds, ratios, timing and filters.
unsigned long long design_hash(const Plan& P)
{
    unsigned long long h = 1469598103934665603ull;
    const int head[4] = {(int) P.passthrough, (int) P.stages.size(), P.trim_stage, P.max_out_len};
    h = fnv(h, head, sizeof head);
    for (const StageDesc& s : P.stages) {
        const int iv[18] = {(int) s.kind, s.up, s.down, s.ref_input_len, s.latency, s.ref_prev_len, (int) s.block_exact,
                            (int) s.is_third, s.in_step, s.out_step, (int) s.fasttiming, s.hb_taps, s.steep_index,
                            s.max_out_len, s.src_history, s.bank.fracs, s.bank.filter_len, s.bank.order};
        const double dv[7] = {s.norm_freq, s.trans_band, s.gain, s.src_rate, s.dst_rate, s.hb_atten, s.bank.atten};
        h = fnv(h, iv, sizeof iv);
        h = fnv(h, dv, sizeof dv);
        h = fnv_v(h, s.lp.taps);
        h = fnv_v(h, s.bank.table);
        h = fnv_v(h, s.hb);
    }
    return h;
}

// Which stage inputs a batch of this plan keeps in shared memory only (fused-away links), and the extra reach of a
// half-band decimator cascade's first stage, as r8bgpu_batch_create decides them when no R8BGPU_* knob is set.
void default_links(const Plan& P, std::vector<char>& fused, std::vector<long long>& extra)
{
    const auto& st = P.stages;
    const size_t ns = st.size();
    fused.assign(ns, 0);
    extra.assign(ns, 0);
    for (size_t i = 0; i < ns; i++) {
        const StageDesc& s = st[i];
        if (plan_fused_stage(st, i, FusedKnobs()).geom.ok) fused[i + 1] = 1;
        if ((s.kind != ST_HBUP && s.kind != ST_HBDOWN) || fused[i]) continue;
        const HbRunPlan hr = plan_hb_run(st, i, HbKnobs());
        const size_t c = (size_t) hr.n_stages;
        if (c < 2) continue;
        if (s.kind == ST_HBDOWN) extra[i] = 2LL * hr.down.back[0] + (2LL << c) + 64;
        for (size_t k = 1; k < c; k++) fused[i + k] = 1;
    }
}

// H_j of every stage input: the longest reach any batch of the plan may re-read below what has arrived -- src_history, plus
// what refilling a fused-away link needs (link_need), plus a decimator cascade's reach -- but no more than the ring a batch
// keeps for a stream that is not fused away.
std::vector<long long> state_windows(const Plan& P)
{
    const auto& st = P.stages;
    const size_t ns = st.size();
    std::vector<char> fused;
    std::vector<long long> extra, need(ns), H(ns);
    default_links(P, fused, extra);
    for (size_t j = ns; j-- > 0;) {
        const StageDesc& s = st[j];
        need[j] = s.src_history + 64;
        if (j + 1 < ns && fused[j + 1]) {
            const long long n = need[j + 1];
            if (s.kind == ST_BLOCKCONV) need[j] += n * s.down / std::max(1, s.up) + 2LL * s.lp.kernel_len + 2;
            else if (s.kind == ST_HBUP) need[j] += n / 2 + s.hb_taps + 2;
            else need[j] += 2 * n + 2LL * s.hb_taps + 2;
        }
    }
    for (size_t j = 0; j < ns; j++) {
        if (fused[j]) {
            H[j] = need[j];
            continue;
        }
        const long long emit_in = j == 0 ? 0 : st[j - 1].max_out_len;
        const long long cap = next_pow2(std::max<long long>(st[j].src_history, extra[j]) + emit_in + 64);
        H[j] = std::min(std::max(need[j], extra[j]), cap);
    }
    return H;
}

size_t header_words(const Plan& P) { return 32 + 8 * P.stages.size(); }

// What an export or import needs of a plan, computed once per plan and call: the design hash walks every filter, and the
// windows re-derive the batch's fusion decisions.
struct PlanState {
    std::vector<long long> H;
    size_t bytes = 0;
    unsigned long long design = 0;
};
thread_local std::map<const Plan*, PlanState>* t_plan_states = nullptr; // set for the duration of one call

const PlanState& plan_state(const Plan& P, PlanState& scratch)
{
    if (t_plan_states != nullptr) {
        auto it = t_plan_states->find(&P);
        if (it != t_plan_states->end()) return it->second;
    }
    PlanState& ps = t_plan_states != nullptr ? (*t_plan_states)[&P] : scratch;
    ps.H = state_windows(P);
    size_t w = header_words(P) + kDitherTaps;
    for (long long h : ps.H) w += (size_t) h;
    ps.bytes = w * 8;
    ps.design = design_hash(P);
    return ps;
}

struct PlanStateScope {
    std::map<const Plan*, PlanState> memo;
    PlanStateScope() { t_plan_states = &memo; }
    ~PlanStateScope() { t_plan_states = nullptr; }
};

size_t state_bytes_of(const Plan& P)
{
    PlanState s;
    return plan_state(P, s).bytes;
}

std::vector<long long> plan_windows(const Plan& P)
{
    PlanState s;
    return plan_state(P, s).H;
}

// The fingerprint words of a header for plan P.
void put_fingerprint(const Plan& P, StateHeader& h)
{
    h.src = P.src_rate;
    h.dst = P.dst_rate;
    h.max_in_len = P.max_in_len;
    h.extfft = P.extfft;
    h.trans_band = P.trans_band;
    h.atten = P.atten;
    h.fasttiming = P.fasttiming;
    h.n_stages = (int32_t) P.stages.size();
    h.max_trim = P.max_trim;
    PlanState s;
    h.design = plan_state(P, s).design;
}

bool same_fingerprint(const Plan& P, const StateHeader& h)
{
    StateHeader f;
    memset(&f, 0, sizeof f);
    put_fingerprint(P, f);
    return memcmp(reinterpret_cast<const char*>(&f) + kFpFirst, reinterpret_cast<const char*>(&h) + kFpFirst, kFpEnd - kFpFirst) == 0;
}

unsigned long long host_terms(const uint64_t* w, size_t n)
{
    unsigned long long s = 0;
    for (size_t i = 0; i < n; i++)
        if (i != 1) s += state_word_term(w[i], i);
    return s;
}

} // namespace

// A plan's channels can move only when they run ragged.
static bool state_plan_ok(const Plan& P, const char* what)
{
    if (!has_fasttiming(P)) return true;
    set_err(std::string(what) + ": R8B_FASTTIMING plans run lock-step only; their streams cannot move");
    return false;
}

static StateStaging& staging_of(r8bgpu_batch* b)
{
    if (!b->stx) b->stx.reset(new StateStaging);
    return *b->stx;
}

// The links that lock-step calls keep in shared memory hold the streams' recent past again (what a ragged call runs first),
// so that a blob does not depend on whether the exporter ran fused or not.  Allocates the link rings if needed.
static bool refill_links(r8bgpu_batch* b, cudaStream_t st)
{
    if (!ensure_ragged_state(b)) return false;
    const size_t ns = b->plan->stages.size();
    bool any = false;
    for (size_t j = 1; j < ns; j++) any = any || b->dev[j].fused_into_prev;
    if (b->links_fresh || !any) {
        b->links_fresh = true;
        return true;
    }
    RaggedRec* h = b->rec.next("refill: records");
    if (h == nullptr) return false;
    std::vector<long long> cnt(ns, 0);
    std::vector<BlockConvParams> bp(ns);
    fill_refill_records(b, channel_schedules(b), h, cnt.data(), bp.data());
    if (!b->rec.upload(0, ns * (size_t) b->n_ch, st, "refill: record upload")) return false;
    refill_launch(b, cnt.data(), bp.data(), st);
    return cuda_ok(cudaGetLastError(), "refill: kernel launch");
}

// Uploads segs and runs one pack / unpack launch over them on st.
static bool run_segments(r8bgpu_batch* b, const std::vector<StateSeg>& segs, long long span, int mode, cudaStream_t st,
                         size_t aux_off = 0)
{
    if (segs.empty() || span <= 0) return true;
    StateStaging& sx = staging_of(b);
    const size_t bytes = segs.size() * sizeof(StateSeg);
    if (!sx.d_aux.grow(b->dev_bytes, aux_off + bytes, "state: cudaMalloc(records)")) return false;
    StateSeg* d = reinterpret_cast<StateSeg*>(sx.d_aux + aux_off);
    if (!cuda_ok(cudaMemcpyAsync(d, segs.data(), bytes, cudaMemcpyHostToDevice, st), "state: record upload") ||
        !cuda_ok(cudaStreamSynchronize(st), "state: record upload"))
        return false;
    if (mode == 0) launch_state_pack(d, (int) segs.size(), span, st);
    else launch_state_unpack(d, (int) segs.size(), span, mode == 1, st);
    b->launches++;
    return cuda_ok(cudaGetLastError(), "state: kernel launch");
}

// The plan channel c of b runs (a mixed batch: its part's).
static const Plan& channel_plan(const r8bgpu_batch* b, int c) { return *slot_of(b, c).b->plan; }

// Packs rows[i] of the ordinary batch b into the device blob dst[i]; the dither setting and history of each stream are
// row drow[i] of `dith` (b's own, or its mixed batch's; null: OFF and empty).  Synchronous.
static bool pack_rows(r8bgpu_batch* b, const std::vector<int>& rows, const std::vector<unsigned char*>& dst,
                      const DitherState* dith, const std::vector<int>& drow)
{
    const Plan& P = *b->plan;
    const size_t ns = P.stages.size(), hw = header_words(P), n = rows.size();
    const std::vector<long long> H = plan_windows(P);
    const size_t bytes = state_bytes_of(P);
    const cudaStream_t st = b->stream;
    if (n == 0) return true;
    if (!cuda_ok(cudaStreamSynchronize(st), "export: sync")) return false;
    if (ns > 0 && !refill_links(b, st)) return false;
    const RaggedSchedule& rs = channel_schedules(b);
    // header words (and a history of zeros where there is no dither state) go in by one launch, the windows by a second
    const size_t row_w = hw + kDitherTaps;
    std::vector<uint64_t> words(n * row_w, 0);
    std::vector<StateSeg> heads(n), segs;
    long long span = 0;
    for (size_t i = 0; i < n; i++) {
        const int r = rows[i];
        uint64_t* w = &words[i * row_w];
        StateHeader h;
        memset(&h, 0, sizeof h);
        h.magic = kStateMagic;
        h.version = kStateVersion;
        h.bytes = bytes;
        put_fingerprint(P, h);
        h.pass_n = b->pass_n[(size_t) r];
        h.trim = b->trim.empty() ? 1.0 : b->trim[(size_t) r];
        if (dith) {
            const DitherCfg& d = dith->cfg[(size_t) drow[i]];
            h.dither_kind = d.kind;
            h.dither_taps = d.n_taps;
            h.dither_seed = d.seed;
            for (int k = 0; k < kDitherTaps; k++) h.taps[k] = d.taps[k];
            h.m = dith->m[(size_t) drow[i]];
        }
        memcpy(w, &h, sizeof h);
        const Schedule& S = rs.of(r);
        long long off = (long long) row_w;
        for (size_t j = 0; j < ns; j++) {
            StateStage g;
            memset(&g, 0, sizeof g);
            g.n_in = S.n_in[j];
            g.n_out = S.n_out[j];
            const Schedule::PolyState& ps = S.poly[j];
            g.in_counter = ps.in_counter;
            g.in_pos_int = ps.in_pos_int;
            g.in_pos_shift = ps.in_pos_shift;
            g.fpos = ps.fpos;
            g.p = ps.p;
            g.dsr = ps.dsr;
            g.window = H[j];
            memcpy(w + 32 + 8 * j, &g, sizeof g);
            const StageDev& d = b->dev[j];
            // what this batch's ring holds of the stream: all of it, or for a fused-away link what the refill rebuilt
            const long long held = d.fused_into_prev ? link_need(b, j) : d.ring_cap;
            StateSeg sg;
            sg.ring = d.ring + (size_t) r * (size_t) d.ring_cap;
            sg.blob = reinterpret_cast<double*>(dst[i]) + off;
            sg.sum = reinterpret_cast<unsigned long long*>(dst[i]) + 1;
            sg.mask = d.ring_cap - 1;
            sg.a0 = S.n_in[j] - H[j];
            sg.len = H[j];
            sg.lo = std::max(0LL, S.n_in[j] - held);
            sg.word0 = off;
            segs.push_back(sg);
            span = std::max(span, sg.len);
            off += H[j];
        }
        if (dith) {
            StateSeg sg;
            sg.ring = dith->d_err + (size_t) drow[i] * kDitherTaps;
            sg.blob = reinterpret_cast<double*>(dst[i]) + hw;
            sg.sum = reinterpret_cast<unsigned long long*>(dst[i]) + 1;
            sg.mask = kDitherTaps - 1;
            sg.a0 = 0;
            sg.len = kDitherTaps;
            sg.lo = 0;
            sg.word0 = (long long) hw;
            segs.push_back(sg);
            span = std::max(span, sg.len);
        }
        w[1] = host_terms(w, dith ? hw : row_w);
        StateSeg& hd = heads[i];
        hd.ring = nullptr; // set below: the uploaded words
        hd.blob = reinterpret_cast<double*>(dst[i]);
        hd.sum = nullptr;
        hd.mask = -1;
        hd.a0 = 0;
        hd.len = (long long) (dith ? hw : row_w);
        hd.lo = 0;
        hd.word0 = 0;
    }
    StateStaging& sx = staging_of(b);
    const size_t wbytes = words.size() * sizeof(uint64_t);
    if (!sx.d_aux.grow(b->dev_bytes, wbytes + heads.size() * sizeof(StateSeg), "export: cudaMalloc(records)")) return false;
    double* dw = reinterpret_cast<double*>((unsigned char*) sx.d_aux);
    if (!cuda_ok(cudaMemcpyAsync(dw, words.data(), wbytes, cudaMemcpyHostToDevice, st), "export: header upload")) return false;
    for (size_t i = 0; i < n; i++) heads[i].ring = dw + i * row_w;
    if (!run_segments(b, heads, (long long) row_w, 0, st, wbytes)) return false;
    // (the window records go behind nothing: the header launch has finished reading its records)
    if (!run_segments(b, segs, span, 0, st)) return false;
    return cuda_ok(cudaStreamSynchronize(st), "export: sync");
}

// Header checks of one blob for channel c of b (hdr: the blob's first header_words() words on the host).
static bool check_header(const r8bgpu_batch* b, int c, const unsigned char* hdr, size_t stride, const char* what)
{
    const Plan& P = channel_plan(b, c);
    const std::string who = std::string(what) + ": channel " + std::to_string(c) + ": ";
    StateHeader h;
    memcpy(&h, hdr, sizeof h);
    if (h.magic != kStateMagic || h.version != kStateVersion) {
        set_err(who + "not a state blob of format version " + std::to_string(kStateVersion));
        return false;
    }
    if (!same_fingerprint(P, h)) {
        if (b->mixed)
            for (const auto& pb : b->mixed->parts)
                if (pb->plan != &P && same_fingerprint(*pb->plan, h)) {
                    set_err(who + "the blob's stream runs another plan of this mixed batch than the channel does");
                    return false;
                }
        set_err(who + "the blob was exported from a batch of a different plan (fingerprint mismatch)");
        return false;
    }
    const size_t size = state_bytes_of(P);
    if (h.bytes != size || stride < size) {
        set_err(who + "truncated blob (" + std::to_string(std::min<size_t>(h.bytes, stride)) + " of " + std::to_string(size) +
                " bytes)");
        return false;
    }
    const std::vector<long long> H = plan_windows(P);
    for (size_t j = 0; j < P.stages.size(); j++) {
        StateStage g;
        memcpy(&g, hdr + sizeof h + j * sizeof g, sizeof g);
        if (g.window != H[j] || g.n_in < 0 || g.n_out < 0) {
            set_err(who + "stage records do not match the plan");
            return false;
        }
    }
    r8bgpu_dither d;
    memset(&d, 0, sizeof d);
    d.kind = h.dither_kind;
    d.n_taps = h.dither_taps;
    d.seed = h.dither_seed;
    for (int k = 0; k < kDitherTaps; k++) d.taps[k] = h.taps[k];
    std::string why;
    if (!dither_cfg_ok(d, why) || h.m < 0 || h.pass_n < 0 ||
        !(P.trim_stage >= 0 ? P.trim_factor_ok(h.trim) : h.trim == 1.0)) {
        set_err(who + "bad stream settings in the blob" + (why.empty() ? std::string() : " (" + why + ")"));
        return false;
    }
    return true;
}

// The checksums of blobs src[i] (device, each with its host header hdr[i]) for channels ch[i] of b, on the device.
static bool check_sums(r8bgpu_batch* b, const std::vector<int>& ch, const std::vector<const unsigned char*>& src,
                       const std::vector<const unsigned char*>& hdr, const char* what)
{
    const size_t n = ch.size();
    if (n == 0) return true;
    StateStaging& sx = staging_of(b);
    const size_t sums_bytes = (n * sizeof(unsigned long long) + 255) & ~(size_t) 255;
    std::vector<StateSeg> segs(n);
    long long span = 0;
    if (!sx.d_aux.grow(b->dev_bytes, sums_bytes + n * sizeof(StateSeg), "import: cudaMalloc(records)")) return false;
    unsigned long long* d_sums = reinterpret_cast<unsigned long long*>((unsigned char*) sx.d_aux);
    for (size_t i = 0; i < n; i++) {
        const Plan& P = channel_plan(b, ch[i]);
        const size_t hw = header_words(P), total = state_bytes_of(P) / 8;
        StateSeg& s = segs[i];
        s.ring = nullptr;
        s.blob = const_cast<double*>(reinterpret_cast<const double*>(src[i])) + hw;
        s.sum = d_sums + i;
        s.mask = -1;
        s.a0 = 0;
        s.len = (long long) (total - hw);
        s.lo = 0;
        s.word0 = (long long) hw;
        span = std::max(span, s.len);
    }
    const cudaStream_t st = b->stream;
    if (!cuda_ok(cudaMemsetAsync(d_sums, 0, n * sizeof(unsigned long long), st), "import: checksum")) return false;
    if (!run_segments(b, segs, span, 1, st, sums_bytes)) return false;
    std::vector<unsigned long long> sums(n);
    if (!cuda_ok(cudaMemcpyAsync(sums.data(), d_sums, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st), "import: checksum") ||
        !cuda_ok(cudaStreamSynchronize(st), "import: checksum"))
        return false;
    for (size_t i = 0; i < n; i++) {
        const size_t hw = header_words(channel_plan(b, ch[i]));
        std::vector<uint64_t> w(hw);
        memcpy(w.data(), hdr[i], hw * 8);
        if (host_terms(w.data(), hw) + sums[i] != w[1]) {
            set_err(std::string(what) + ": channel " + std::to_string(ch[i]) + ": bad checksum (the blob is damaged)");
            return false;
        }
    }
    return true;
}

// Installs blobs src[i] (device, verified; hdr[i] on the host) as the streams of rows[i] of the ordinary batch b.
static bool unpack_rows(r8bgpu_batch* b, const std::vector<int>& rows, const std::vector<const unsigned char*>& src,
                        const std::vector<const unsigned char*>& hdr)
{
    const Plan& P = *b->plan;
    const size_t ns = P.stages.size(), hw = header_words(P), n = rows.size();
    const cudaStream_t st = b->stream;
    if (n == 0) return true;
    if (!cuda_ok(cudaStreamSynchronize(st), "import: sync")) return false;
    // the batch's own channels first get their links back, so the imported windows are the only ones not recomputed
    if (ns > 0 && !refill_links(b, st)) return false;
    std::vector<Schedule> sched(n);
    std::vector<StateSeg> segs;
    long long span = 0;
    for (size_t i = 0; i < n; i++) {
        StateHeader h;
        memcpy(&h, hdr[i], sizeof h);
        Schedule& S = sched[i];
        S.init(b->plan);
        long long off = (long long) (hw + kDitherTaps);
        for (size_t j = 0; j < ns; j++) {
            StateStage g;
            memcpy(&g, hdr[i] + sizeof h + j * sizeof g, sizeof g);
            S.n_in[j] = g.n_in;
            S.n_out[j] = g.n_out;
            Schedule::PolyState& ps = S.poly[j];
            ps.in_counter = g.in_counter;
            ps.in_pos_int = g.in_pos_int;
            ps.in_pos_shift = g.in_pos_shift;
            ps.fpos = g.fpos;
            ps.p = g.p;
            ps.dsr = g.dsr;
            const StageDev& d = b->dev[j];
            StateSeg sg;
            sg.ring = d.ring + (size_t) rows[i] * (size_t) d.ring_cap;
            sg.blob = const_cast<double*>(reinterpret_cast<const double*>(src[i])) + off;
            sg.sum = nullptr;
            sg.mask = d.ring_cap - 1;
            sg.a0 = g.n_in - g.window;
            sg.len = g.window;
            sg.lo = 0;
            sg.word0 = off;
            segs.push_back(sg);
            span = std::max(span, d.ring_cap);
            off += g.window;
        }
        b->pass_n[(size_t) rows[i]] = h.pass_n;
        if (!b->trim.empty()) b->trim[(size_t) rows[i]] = h.trim;
    }
    if (!run_segments(b, segs, span, 2, st)) return false;
    channel_schedules(b);
    b->rag.install(rows.data(), (int) n, sched.data());
    b->diverged = !b->rag.converged();
    if (!b->diverged) b->sched = b->rag.groups[0];
    return cuda_ok(cudaStreamSynchronize(st), "import: sync");
}

// The dither settings and histories of the blobs become those of channels ch[i] of b (ordinary or mixed: the batch that
// owns the conversions into the caller's buffers).
static bool unpack_dither(r8bgpu_batch* b, const std::vector<int>& ch, const std::vector<const unsigned char*>& src,
                          const std::vector<const unsigned char*>& hdr)
{
    const size_t n = ch.size();
    std::vector<r8bgpu_dither> cfg(n);
    bool need = b->dith != nullptr;
    for (size_t i = 0; i < n; i++) {
        StateHeader h;
        memcpy(&h, hdr[i], sizeof h);
        r8bgpu_dither& d = cfg[i];
        memset(&d, 0, sizeof d);
        d.kind = h.dither_kind;
        d.n_taps = h.dither_taps;
        d.seed = h.dither_seed;
        for (int k = 0; k < kDitherTaps; k++) d.taps[k] = h.taps[k];
        need = need || d.kind != R8BGPU_DITHER_OFF || h.m != 0;
    }
    if (!need || n == 0) return true;
    if (r8bgpu_batch_set_dither(b, ch.data(), (int) n, cfg.data()) != 0) return false;
    std::vector<StateSeg> segs(n);
    for (size_t i = 0; i < n; i++) {
        StateHeader h;
        memcpy(&h, hdr[i], sizeof h);
        b->dith->m[(size_t) ch[i]] = h.m;
        const size_t hw = header_words(channel_plan(b, ch[i]));
        StateSeg& s = segs[i];
        s.ring = b->dith->d_err + (size_t) ch[i] * kDitherTaps;
        s.blob = const_cast<double*>(reinterpret_cast<const double*>(src[i])) + hw;
        s.sum = nullptr;
        s.mask = kDitherTaps - 1;
        s.a0 = 0;
        s.len = kDitherTaps;
        s.lo = 0;
        s.word0 = (long long) hw;
    }
    return run_segments(b, segs, kDitherTaps, 2, b->stream) && cuda_ok(cudaStreamSynchronize(b->stream), "import: sync");
}

// Channels, plans and buffer of an export or import, checked before anything happens.  jobs: the batches that hold the
// named streams' device state, with their rows -- a front's shards, else b itself (a mixed batch reaches its parts in
// export_dev / import_dev, since it keeps the streams' dither state).
static bool check_state_call(r8bgpu_batch* b, const int* channels, int n, const void* buf, size_t stride, bool device,
                             const char* what, std::vector<ChannelGroup>& jobs)
{
    if (b == nullptr || n < 0 || (n > 0 && (channels == nullptr || buf == nullptr))) {
        set_err(std::string(what) + ": bad arguments");
        return false;
    }
    if (device && b->front) {
        set_err(std::string(what) + ": device buffers live on one GPU; move the streams of a multi-device batch through host "
                "memory, or call its shards (r8bgpu_batch_shard())");
        return false;
    }
    if (device && (stride % 8 != 0 || reinterpret_cast<uintptr_t>(buf) % 8 != 0)) {
        set_err(std::string(what) + ": device blobs must be 8-byte aligned (buf and stride_bytes)");
        return false;
    }
    const bool ok = check_channels(b, channels, n, what, true, [&](int, int c) {
        const Plan& P = channel_plan(b, c);
        if (!state_plan_ok(P, what)) return false;
        if (stride < state_bytes_of(P)) {
            set_err(std::string(what) + ": stride_bytes " + std::to_string(stride) + " is smaller than channel " +
                    std::to_string(c) + "'s blob (" + std::to_string(state_bytes_of(P)) + " bytes)");
            return false;
        }
        return true;
    });
    if (!ok) return false;
    if (b->front) {
        jobs = group_channels(b, channels, n);
    } else {
        jobs.assign(1, ChannelGroup{b, std::vector<int>(channels, channels + n), {}});
        for (int i = 0; i < n; i++) jobs[0].idx.push_back(i);
    }
    return true;
}

// Exports channels ch of the ordinary or mixed batch b into the device blobs dst[i].
static bool export_dev(r8bgpu_batch* b, const std::vector<int>& ch, const std::vector<unsigned char*>& dst)
{
    if (!b->mixed) return pack_rows(b, ch, dst, b->dith.get(), ch);
    // (conversions queued on the batch stream may still update the dither histories)
    if (!cuda_ok(cudaStreamSynchronize(b->stream), "export: sync")) return false;
    for (const ChannelGroup& G : group_channels(b, ch.data(), (int) ch.size()))
        if (!pack_rows(G.b, G.rows, gather(dst.data(), G.idx), b->dith.get(), gather(ch.data(), G.idx))) return false;
    return true;
}

// Imports device blobs src[i] (host headers hdr[i], verified) into channels ch of the ordinary or mixed batch b.
static bool import_dev(r8bgpu_batch* b, const std::vector<int>& ch, const std::vector<const unsigned char*>& src,
                       const std::vector<const unsigned char*>& hdr)
{
    if (!b->mixed) return unpack_rows(b, ch, src, hdr) && unpack_dither(b, ch, src, hdr);
    for (const ChannelGroup& G : group_channels(b, ch.data(), (int) ch.size()))
        if (!unpack_rows(G.b, G.rows, gather(src.data(), G.idx), gather(hdr.data(), G.idx))) return false;
    return unpack_dither(b, ch, src, hdr);
}

static int state_export(r8bgpu_batch* b, const int* channels, int n, void* buf, size_t stride, bool device)
{
    const char* what = device ? "batch_export_device" : "batch_export";
    PlanStateScope scope;
    std::vector<ChannelGroup> jobs;
    if (!check_state_call(b, channels, n, buf, stride, device, what, jobs)) return -1;
    for (const ChannelGroup& J : jobs) {
        if (J.rows.empty()) continue;
        DeviceGuard g(J.b->device);
        std::vector<unsigned char*> dst(J.rows.size());
        if (device) {
            for (size_t i = 0; i < J.rows.size(); i++) dst[i] = static_cast<unsigned char*>(buf) + (size_t) J.idx[i] * stride;
            if (!export_dev(J.b, J.rows, dst)) return -1;
            continue;
        }
        // host form: the device form into staging, then one copy over PCIe into pinned memory, then the caller's rows
        size_t w = 0;
        for (int c : J.rows) w = std::max(w, state_bytes_of(channel_plan(J.b, c)));
        StateStaging& sx = staging_of(J.b);
        if (!sx.d_blob.grow(J.b->dev_bytes, w * J.rows.size(), "export: cudaMalloc(staging)") ||
            !sx.h_blob.grow(w * J.rows.size(), "state: cudaMallocHost"))
            return -1;
        for (size_t i = 0; i < J.rows.size(); i++) dst[i] = sx.d_blob + i * w;
        if (!export_dev(J.b, J.rows, dst)) return -1;
        if (!cuda_ok(cudaMemcpy(sx.h_blob, sx.d_blob, w * J.rows.size(), cudaMemcpyDeviceToHost), "export: copy to host")) return -1;
        for (size_t i = 0; i < J.rows.size(); i++)
            memcpy(static_cast<unsigned char*>(buf) + (size_t) J.idx[i] * stride, sx.h_blob + i * w,
                   state_bytes_of(channel_plan(J.b, J.rows[i])));
    }
    return 0;
}

static int state_import(r8bgpu_batch* b, const int* channels, int n, const void* buf, size_t stride, bool device)
{
    const char* what = device ? "batch_import_device" : "batch_import";
    PlanStateScope scope;
    std::vector<ChannelGroup> jobs;
    if (!check_state_call(b, channels, n, buf, stride, device, what, jobs)) return -1;
    // every blob is checked, on every shard, before any channel changes: a refused call changes nothing
    std::vector<std::vector<unsigned char>> hdr_store(jobs.size());
    std::vector<std::vector<const unsigned char*>> src(jobs.size()), hdr(jobs.size());
    for (size_t k = 0; k < jobs.size(); k++) {
        const ChannelGroup& J = jobs[k];
        if (J.rows.empty()) continue;
        DeviceGuard g(J.b->device);
        const size_t m = J.rows.size();
        size_t hb = 0, w = 0;
        for (int c : J.rows) {
            hb = std::max(hb, header_words(channel_plan(J.b, c)) * 8);
            w = std::max(w, state_bytes_of(channel_plan(J.b, c)));
        }
        src[k].resize(m);
        hdr[k].resize(m);
        if (device) {
            // the headers cross PCIe; the windows stay where they are
            hdr_store[k].resize(m * hb);
            for (size_t i = 0; i < m; i++) {
                src[k][i] = static_cast<const unsigned char*>(buf) + (size_t) J.idx[i] * stride;
                if (!cuda_ok(cudaMemcpy(hdr_store[k].data() + i * hb, src[k][i], hb, cudaMemcpyDeviceToHost), "import: headers"))
                    return -1;
                hdr[k][i] = hdr_store[k].data() + i * hb;
            }
        } else {
            for (size_t i = 0; i < m; i++) hdr[k][i] = static_cast<const unsigned char*>(buf) + (size_t) J.idx[i] * stride;
        }
        for (size_t i = 0; i < m; i++)
            if (!check_header(J.b, J.rows[i], hdr[k][i], stride, what)) return -1;
        if (!device) {
            StateStaging& sx = staging_of(J.b);
            if (!sx.d_blob.grow(J.b->dev_bytes, w * m, "import: cudaMalloc(staging)") ||
                !sx.h_blob.grow(w * m, "state: cudaMallocHost"))
                return -1;
            for (size_t i = 0; i < m; i++) {
                memcpy(sx.h_blob + i * w, hdr[k][i], state_bytes_of(channel_plan(J.b, J.rows[i])));
                src[k][i] = sx.d_blob + i * w;
            }
            if (!cuda_ok(cudaMemcpy(sx.d_blob, sx.h_blob, w * m, cudaMemcpyHostToDevice), "import: copy to device")) return -1;
        }
        if (!check_sums(J.b, J.rows, src[k], hdr[k], what)) return -1;
    }
    for (size_t k = 0; k < jobs.size(); k++) {
        if (jobs[k].rows.empty()) continue;
        DeviceGuard g(jobs[k].b->device);
        if (!import_dev(jobs[k].b, jobs[k].rows, src[k], hdr[k])) return -1;
    }
    return 0;
}

extern "C" {

size_t r8bgpu_plan_state_bytes(const r8bgpu_plan* plan) { return plan ? state_bytes_of(plan->p) : 0; }

int r8bgpu_plan_state_windows(const r8bgpu_plan* plan, long long* windows, int cap)
{
    if (plan == nullptr) {
        set_err("plan_state_windows: null plan");
        return -1;
    }
    const std::vector<long long> H = state_windows(plan->p);
    for (size_t j = 0; j < H.size() && (int) j < cap; j++)
        if (windows != nullptr) windows[j] = H[j];
    return (int) H.size();
}

int r8bgpu_plan_state_fingerprint(const r8bgpu_plan* plan, void* out, int cap)
{
    if (plan == nullptr) {
        set_err("plan_state_fingerprint: null plan");
        return -1;
    }
    StateHeader h;
    memset(&h, 0, sizeof h);
    put_fingerprint(plan->p, h);
    const int n = (int) (kFpEnd - kFpFirst);
    if (out != nullptr) memcpy(out, reinterpret_cast<const char*>(&h) + kFpFirst, (size_t) std::min(n, cap));
    return n;
}

// The blob (format version 1) carries no modulator state: a stream with DSD output cannot move.
static bool refuse_dsd_state(const r8bgpu_batch* b, const char* what)
{
    if (!dsd_on(b)) return false;
    set_err(std::string(what) + ": DSD output is on (r8bgpu_batch_set_dsd_out); the state blob does not carry the modulators' "
            "state: turn it off first");
    return true;
}

int r8bgpu_batch_export(r8bgpu_batch* b, const int* channels, int n, void* buf, size_t stride_bytes)
{
    if (refuse_dsd_state(b, "batch_export")) return -1;
    return state_export(b, channels, n, buf, stride_bytes, false);
}

int r8bgpu_batch_import(r8bgpu_batch* b, const int* channels, int n, const void* buf, size_t stride_bytes)
{
    if (refuse_dsd_state(b, "batch_import")) return -1;
    return state_import(b, channels, n, buf, stride_bytes, false);
}

int r8bgpu_batch_export_device(r8bgpu_batch* b, const int* channels, int n, void* buf, size_t stride_bytes)
{
    if (refuse_dsd_state(b, "batch_export_device")) return -1;
    return state_export(b, channels, n, buf, stride_bytes, true);
}

int r8bgpu_batch_import_device(r8bgpu_batch* b, const int* channels, int n, const void* buf, size_t stride_bytes)
{
    if (refuse_dsd_state(b, "batch_import_device")) return -1;
    return state_import(b, channels, n, buf, stride_bytes, true);
}

// ---- long clips: whole clips cut into warm-started segments, one per lane (include/r8bgpu.h, "long clips") -----------

// W before rounding (DESIGN.md section 10).  Stream j is the input of stage j; lane samples below S are zeros where the
// twin has its input.  t_j: the first index of stream j from which the lane's values are the twin's bits; n_j(P): the
// twin's total of stream j after P source samples.  Each stage bounds both by lines in its input:
//   t_{j+1} <= rho t_j + beta   (an output is exact once everything its kernel mixes into it is exact)
//   n_{j+1} >= rho n_j - gamma  (the emission lower bounds of flush_max_out_len)
//   BlockConv (U, D): an output of an overlap-save tile mixes the rounding of the whole tile, and tiles are transformed
//              in pairs (two real tiles in one complex FFT), so of 2 M tile samples (at least one per input sample, M the
//              largest tile a ragged call may use), reaching K taps behind its position:
//              beta = (U (2 M + 2) + K) / D + 2, gamma = Latency / D + 1.
//   Frac:      output q reads [p_q - fll, p_q - fll + flen), p_q >= q / rho - 2: beta = (fll + 3) rho + 2.
//   HBUp:      output 2n + 1 reads [n - T + 1, n + T]: beta = 2 T + 4.      HBDown: [2m - 2T + 1, 2m + 2T - 1]: beta = T + 2.
// With r_j the product of the ratios in front of stage j, t_j <= r_j S + c_j and n_j(P) >= r_j P - C_j, so the window
// [n_j - reach_j, n_j) a later call can re-read (reach_j: the larger of H_j and src_history + 64) holds exact bits when
// r_j (P - S) >= c_j + C_j + reach_j for every j.
static long long oneshot_warmup_raw(const Plan& P)
{
    if (P.passthrough) return 0;
    const std::vector<long long> H = plan_windows(P);
    double r = 1.0, c = 0.0, C = 0.0, w = 0.0;
    for (size_t j = 0; j < P.stages.size(); j++) {
        const StageDesc& s = P.stages[j];
        const double reach = (double) std::max(H[j], (long long) s.src_history + 64);
        w = std::max(w, (c + C + reach) / r);
        double rho = 1.0, beta = 0.0, gamma = 0.0;
        switch (s.kind) {
        case ST_BLOCKCONV: {
            const BcTile t = blockconv_tile(s, true);
            const double M = (double) std::max(1 << std::max(t.fft_log2, 0), 4096);
            rho = (double) s.up / s.down;
            beta = ((double) s.up * (2.0 * M + 2.0) + s.lp.kernel_len) / s.down + 2.0;
            gamma = (double) s.latency / s.down + 1.0;
            break;
        }
        case ST_FRAC_WHOLE:
        case ST_FRAC_POLY: {
            rho = s.kind == ST_FRAC_WHOLE ? (double) s.out_step / s.in_step : s.dst_rate / s.src_rate;
            const double fll = s.bank.filter_len / 2 - 1;
            beta = (fll + 3.0) * rho + 2.0;
            gamma = (s.bank.filter_len / 2 + 2) * rho + 2.0;
            break;
        }
        case ST_HBUP:
            rho = 2.0;
            beta = 2.0 * s.hb_taps + 4.0;
            gamma = 2.0 * s.hb_taps + 2.0;
            break;
        case ST_HBDOWN:
            rho = 0.5;
            beta = s.hb_taps + 2.0;
            gamma = s.hb_taps + 1.0;
            break;
        }
        c = rho * c + beta;
        C = rho * C + gamma;
        r *= rho;
    }
    return (long long) std::ceil(w) + 1;
}

// W in blocks of MaxInLen: enough whole blocks even where DSD input shortens the block to a multiple of 8
static long long oneshot_warmup_blocks(const Plan& P)
{
    const long long raw = oneshot_warmup_raw(P);
    const long long b = P.max_in_len >= 8 ? P.max_in_len & ~7LL : P.max_in_len;
    return (raw + b - 1) / b;
}

static const char* oneshot_plan_refusal(const Plan& P)
{
    if (P.trim_stage >= 0) return "trim plans run a per-channel factor; long clips run the plan's own ratio";
    if (has_fasttiming(P)) return "R8B_FASTTIMING plans run lock-step only (their positions drift sequentially)";
    return nullptr;
}

// The segments of a call (policy: include/r8bgpu.h, "long clips"), by round and lane; start[i] (states: non-null) is the
// twin's schedule at segs[i].start, and seg_flush[i] says that segs[i] ends in its clip's flush.  calls[r]: the block
// calls of round r; flush[r]: the round ends with a flush.
struct OneshotLayout {
    std::vector<r8bgpu_oneshot_seg> segs;
    std::vector<Schedule> start;
    std::vector<char> seg_flush;
    std::vector<long long> calls;
    std::vector<char> flush;
    long long n_calls = 0;
};

// A stretch of one clip's twin run that a call keeps: the outputs [e0, e1) of the blocks [b0, b1) of clip `clip`, and with
// `flush` the twin's flush to its oplens after them.  row: the output row (the clip for whole clips, the crop for crops),
// whose element 0 is output e0 of a crop and output 0 of a whole clip.  A whole clip is the span (0, nb, 0, oplen, flush).
struct OneshotSpan {
    int clip, row;
    long long b0, b1, e0, e1;
    bool flush;
};

// The whole clips r of idx as spans (rows: the clips themselves)
static std::vector<OneshotSpan> oneshot_clip_spans(long long B, const std::vector<int>& idx, const long long* lens,
                                                   const long long* oplens)
{
    std::vector<OneshotSpan> sp;
    for (int r : idx) sp.push_back(OneshotSpan{r, r, 0, (lens[r] + B - 1) / B, 0, oplens[r], true});
    return sp;
}

// Segments are cut from each span's first block by the long-clip policy; segs[i].clip is the index of its span.  Every
// clip's twin is walked once, however many spans name it.
static void oneshot_layout(const Plan& P, long long B, int n_lanes, const std::vector<OneshotSpan>& spans, const long long* lens,
                           bool states, OneshotLayout& L)
{
    const long long wb = oneshot_warmup_blocks(P);
    const size_t n_spans = spans.size();
    std::vector<long long> nb(n_spans);
    long long m = 0, nb_max = 1;
    for (size_t i = 0; i < n_spans; i++) {
        nb[i] = spans[i].b1 - spans[i].b0;
        if (spans[i].e1 > spans[i].e0) m++;
        nb_max = std::max(nb_max, nb[i]);
    }
    const long long lanes = std::max(1LL, (m + n_lanes - 1) / n_lanes) * n_lanes;
    auto count = [&](long long len_blocks) {
        long long n = 0;
        for (size_t i = 0; i < n_spans; i++)
            if (spans[i].e1 > spans[i].e0) n += std::max(1LL, (nb[i] + len_blocks - 1) / len_blocks);
        return n;
    };
    long long lo = 0, hi = nb_max; // count(hi) <= lanes; find the fewest blocks per segment that fits
    while (hi - lo > 1) {
        const long long mid = lo + (hi - lo) / 2;
        (count(mid) <= lanes ? hi : lo) = mid;
    }
    const long long seg_blocks = hi;
    struct Item {
        r8bgpu_oneshot_seg s;
        long long cost;
        bool last; // the span's last segment, and the span ends in the flush
        Schedule st;
    };
    // the spans of each clip, in span order
    std::map<int, std::vector<size_t>> by_clip;
    for (size_t i = 0; i < n_spans; i++)
        if (spans[i].e1 > spans[i].e0) by_clip[spans[i].clip].push_back(i);
    std::vector<std::vector<Item>> per_span(n_spans);
    std::vector<StageCall> calls;
    for (const auto& kv : by_clip) {
        const long long len = lens[kv.first];
        // walk the twin once: its output total at every block boundary up to the last one a span needs, and its schedule
        // at every S_k
        long long top = 0;
        std::map<long long, Schedule> snap; // block index -> schedule
        for (size_t i : kv.second) {
            const OneshotSpan& sp = spans[i];
            top = std::max(top, sp.b1);
            const long long K = std::max(1LL, (nb[i] + seg_blocks - 1) / seg_blocks);
            for (long long k = 0; k < K; k++) snap[std::max(0LL, sp.b0 + k * seg_blocks - wb)] = Schedule();
        }
        std::vector<long long> E((size_t) top + 1, 0);
        Schedule s;
        s.init(&P);
        for (long long blk = 0;; blk++) {
            const long long pos = std::min(blk * B, len);
            E[(size_t) blk] = P.passthrough ? pos : s.outputs();
            auto it = snap.find(blk);
            if (states && it != snap.end()) it->second = s;
            if (blk >= top) break;
            s.advance((int) std::min(B, len - pos), calls);
        }
        for (size_t i : kv.second) {
            const OneshotSpan& sp = spans[i];
            const long long K = std::max(1LL, (nb[i] + seg_blocks - 1) / seg_blocks);
            auto kept = [&](long long e) { return std::min(std::max(e, sp.e0), sp.e1); };
            for (long long k = 0; k < K; k++) {
                const long long b0 = sp.b0 + k * seg_blocks, b1 = std::min(b0 + seg_blocks, sp.b1);
                Item it;
                it.s.clip = (int) i;
                it.s.p0 = b0 * B;
                it.s.p1 = std::min(b1 * B, len);
                it.s.start = std::max(0LL, it.s.p0 - wb * B);
                it.last = k + 1 == K && sp.flush;
                it.s.e0 = kept(E[(size_t) b0]);
                it.s.e1 = it.last ? sp.e1 : kept(E[(size_t) b1]);
                it.s.pad_ = 0;
                if (it.s.e1 <= it.s.e0) continue;
                it.cost = (it.s.p1 - it.s.start + B - 1) / B;
                if (states) it.st = snap[it.s.start / B];
                per_span[i].push_back(std::move(it));
            }
        }
    }
    std::vector<Item> items;
    for (auto& v : per_span)
        for (Item& it : v) items.push_back(std::move(it));
    std::stable_sort(items.begin(), items.end(), [](const Item& a, const Item& b) { return a.cost > b.cost; });
    L = OneshotLayout();
    for (size_t i = 0; i < items.size(); i++) {
        const int round = (int) (i / (size_t) n_lanes);
        if ((size_t) round == L.calls.size()) {
            L.calls.push_back(0);
            L.flush.push_back(0);
        }
        L.calls[(size_t) round] = std::max(L.calls[(size_t) round], items[i].cost);
        if (items[i].last) L.flush[(size_t) round] = 1;
        r8bgpu_oneshot_seg g = items[i].s;
        g.round = round;
        g.lane = (int) (i % (size_t) n_lanes);
        L.segs.push_back(g);
        L.seg_flush.push_back(items[i].last ? 1 : 0);
        if (states) L.start.push_back(std::move(items[i].st));
    }
    for (size_t k = 0; k < L.calls.size(); k++) L.n_calls += L.calls[k] + L.flush[k];
}

// The spans of crops (include/r8bgpu.h, "crops of long clips"): crop k of the list (clip c, outputs [o0, o1)) starts at
// P_lo, the first block boundary below lens[c] (or 0) whose E is the largest E <= o0 (so a crop from output 0 starts at
// 0, as the whole clip does, however many blocks the latency takes), and ends at the first block boundary (or lens[c])
// with E >= o1, or, when o1 > E(lens[c]), in the twin's flush to oplens[c].  Row: crop k.  One walk per clip, whatever
// its crop count, up to the boundary that its last-ending crop needs.
static std::vector<OneshotSpan> oneshot_crop_spans(const Plan& P, long long B, const std::vector<int>& ks, const r8bgpu_crop* crops,
                                                   const long long* lens)
{
    std::vector<OneshotSpan> sp(ks.size());
    std::map<int, std::vector<size_t>> by_clip;
    for (size_t i = 0; i < ks.size(); i++) by_clip[crops[ks[i]].clip].push_back(i);
    std::vector<StageCall> calls;
    for (const auto& kv : by_clip) {
        const long long len = lens[kv.first], nb = (len + B - 1) / B;
        long long need = 0;
        for (size_t i : kv.second) need = std::max(need, crops[ks[i]].o1);
        std::vector<long long> E; // E[blk]: the twin's output total after min(blk B, len) inputs
        Schedule s;
        s.init(&P);
        for (long long blk = 0;; blk++) {
            const long long pos = std::min(blk * B, len);
            E.push_back(P.passthrough ? pos : s.outputs());
            if (blk >= nb || E.back() >= need) break;
            s.advance((int) std::min(B, len - pos), calls);
        }
        const long long top = (long long) E.size() - 1; // E is complete up to here; E(len) < need when top == nb
        for (size_t i : kv.second) {
            const r8bgpu_crop& c = crops[ks[i]];
            OneshotSpan& o = sp[i];
            o.clip = c.clip;
            o.row = ks[i];
            o.e0 = c.o0;
            o.e1 = c.o1;
            // P_lo: a block boundary before the clip's end, so that S = P_lo - W is one too
            const long long b0_max = std::max(0LL, std::min(nb - 1, top));
            o.b0 = (long long) (std::upper_bound(E.begin(), E.begin() + b0_max + 1, c.o0) - E.begin()) - 1;
            o.b0 = std::max(0LL, o.b0);
            while (o.b0 > 0 && E[(size_t) o.b0 - 1] == E[(size_t) o.b0]) o.b0--; // of blocks with no output, the first
            const long long b1 = (long long) (std::lower_bound(E.begin() + o.b0, E.end(), c.o1) - E.begin());
            o.flush = b1 > top; // no boundary reaches o1: top == nb and E(len) < o1
            o.b1 = o.flush ? nb : b1;
        }
    }
    return sp;
}

// A long-clip call checked and normalised: clip r runs *plan[r] to its flush target op[r].  The output rows are the
// clips (op[r] samples each) or, with crops, the crops (o1 - o0 samples each); rows[p] holds part p's rows, ascending.
struct OneshotCall {
    bool cropped = false;
    const r8bgpu_crop* crops = nullptr;
    std::vector<const Plan*> plan;
    std::vector<long long> op, row_len;
    std::vector<std::vector<int>> rows;
    std::string row_kind() const { return cropped ? "crop" : "clip"; }
};

// The checks every long-clip call shares, in this order: lengths, plan indices, plan refusals, targets, crops.  parts:
// the plan of each part (an ordinary batch, or a plan alone: one part); mixed: a mixed batch, whose parts are judged
// only when they have rows and are named in the refusal.  A NULL plan_of_clip is all zeros, except on a mixed batch.
// Messages start with w, those of plan indices with w_idx.
static bool oneshot_call(const std::string& w, const std::string& w_idx, const std::vector<const Plan*>& parts, bool mixed,
                         int n_clips, const int* plan_of_clip, const long long* lens, const long long* oplens, bool cropped,
                         int n_crops, const r8bgpu_crop* crops, OneshotCall& c)
{
    auto fail = [&](const std::string& m) {
        set_err(w + ": " + m);
        return false;
    };
    auto fail_idx = [&](const std::string& m) {
        set_err(w_idx + ": " + m);
        return false;
    };
    if (n_clips < 0 || (n_clips > 0 && lens == nullptr)) return fail("bad arguments");
    for (int r = 0; r < n_clips; r++)
        if (lens[r] < 0 || (oplens != nullptr && oplens[r] < 0)) return fail("negative length (clip " + std::to_string(r) + ")");
    if (mixed && n_clips > 0 && plan_of_clip == nullptr) return fail_idx("null plan_of_clip");
    const int np = (int) parts.size();
    c = OneshotCall();
    c.cropped = cropped;
    c.crops = crops;
    c.rows.assign((size_t) np, std::vector<int>());
    std::vector<int> part((size_t) n_clips, 0);
    for (int r = 0; r < n_clips; r++) {
        const int p = plan_of_clip != nullptr ? plan_of_clip[r] : 0;
        if (p < 0 || p >= np)
            return fail_idx("plan_of_clip[" + std::to_string(r) + "] = " + std::to_string(p) + " is not a plan index of the batch (" +
                            std::to_string(np) + " plans)");
        part[(size_t) r] = p;
        c.plan.push_back(parts[(size_t) p]);
        if (!cropped) c.rows[(size_t) p].push_back(r);
    }
    for (int k = 0; cropped && crops != nullptr && k < n_crops; k++)
        if (crops[k].clip >= 0 && crops[k].clip < n_clips) c.rows[(size_t) part[(size_t) crops[k].clip]].push_back(k);
    for (int p = 0; p < np; p++)
        if (!mixed || !c.rows[(size_t) p].empty())
            if (const char* why = oneshot_plan_refusal(*parts[(size_t) p]))
                return fail((mixed ? "plans[" + std::to_string(p) + "]: " : std::string()) + why);
    for (int r = 0; r < n_clips; r++) {
        c.op.push_back(oplens != nullptr ? oplens[r] : flush_default_target(*c.plan[(size_t) r], lens[r]));
        if (c.op.back() < 0) return fail("the default output length does not fit a long long");
    }
    if (!cropped) {
        c.row_len = c.op;
        return true;
    }
    // crops: refused, naming the crop, where no twin run holds them
    if (n_crops < 0) return fail("bad arguments");
    if (n_crops > 0 && crops == nullptr) return fail("null crops");
    for (int k = 0; k < n_crops; k++) {
        const r8bgpu_crop& q = crops[k];
        const std::string at = "crops[" + std::to_string(k) + "]";
        if (q.clip < 0 || q.clip >= n_clips)
            return fail(at + ".clip = " + std::to_string(q.clip) + " is not a clip of the call (" + std::to_string(n_clips) + " clips)");
        if (q.o0 < 0) return fail(at + ".o0 = " + std::to_string(q.o0) + " is negative");
        if (q.o1 < q.o0) return fail(at + ".o1 = " + std::to_string(q.o1) + " is before o0 = " + std::to_string(q.o0));
        if (q.o1 > c.op[(size_t) q.clip])
            return fail(at + ".o1 = " + std::to_string(q.o1) + " is past oplens[" + std::to_string(q.clip) +
                        "] = " + std::to_string(c.op[(size_t) q.clip]));
        c.row_len.push_back(q.o1 - q.o0);
    }
    return true;
}

// The spans of part p's rows: its whole clips, or its crops
static std::vector<OneshotSpan> oneshot_spans(const Plan& P, long long B, const OneshotCall& c, size_t p, const long long* lens)
{
    return c.cropped ? oneshot_crop_spans(P, B, c.rows[p], c.crops, lens) : oneshot_clip_spans(B, c.rows[p], lens, c.op.data());
}

long long r8bgpu_plan_oneshot_warmup(const r8bgpu_plan* plan)
{
    return plan == nullptr ? -1 : oneshot_warmup_blocks(plan->p) * plan->p.max_in_len;
}

// The dry runs (r8bgpu_plan_simulate_oneshot / _simulate_oneshot_crops): the layout a call of plan on n_lanes lanes runs
static int oneshot_simulate(const char* what, const r8bgpu_plan* plan, int n_lanes, int n_clips, const long long* lens,
                            const long long* oplens, bool cropped, int n_crops, const r8bgpu_crop* crops, int* n_calls,
                            r8bgpu_oneshot_seg* seg, int cap)
{
    if (plan == nullptr || n_lanes < 1) {
        set_err(std::string(what) + ": bad arguments");
        return -1;
    }
    const Plan& P = plan->p;
    OneshotCall c;
    if (!oneshot_call(what, what, {&P}, false, n_clips, nullptr, lens, oplens, cropped, n_crops, crops, c)) return -1;
    OneshotLayout L;
    oneshot_layout(P, P.max_in_len, n_lanes, oneshot_spans(P, P.max_in_len, c, 0, lens), lens, false, L);
    if (n_calls != nullptr) *n_calls = (int) std::min<long long>(L.n_calls, INT_MAX);
    for (size_t i = 0; seg != nullptr && i < L.segs.size() && (int) i < cap; i++) seg[i] = L.segs[i];
    return (int) L.segs.size();
}

int r8bgpu_plan_simulate_oneshot(const r8bgpu_plan* plan, int n_lanes, int n_clips, const long long* lens,
                                 const long long* oplens, int* n_calls, r8bgpu_oneshot_seg* seg, int cap)
{
    return oneshot_simulate("plan_simulate_oneshot", plan, n_lanes, n_clips, lens, oplens, false, 0, nullptr, n_calls, seg, cap);
}

// The buffers of a checked long-clip call: the input holds its clips, the output its rows; every check runs before
// anything changes.  out: the block length B.
static bool oneshot_args(const std::string& w, const r8bgpu_batch* b, const r8bgpu_buffer& in, const r8bgpu_buffer& out,
                         const OneshotCall& c, const long long* lens, const r8bgpu_dither* dither, long long& B)
{
    auto fail = [&](const std::string& m) {
        set_err(w + ": " + m);
        return false;
    };
    const int n_clips = (int) c.plan.size();
    if (dsd_on(b)) return fail("DSD output is on: its modulators run sequentially through a whole clip");
    const FormatElem fi = format_elem(in.format), fo = format_elem(out.format);
    if (fi.bytes == 0 || fo.bytes == 0) return fail("unknown sample format");
    if (is_dsd_format(out.format)) return fail("DSD formats are input-only here");
    if (!(in.scale == in.scale) || in.scale == 0.0 || !(out.scale == out.scale) || out.scale == 0.0)
        return fail("scale must be a non-zero number");
    for (int r = 0; dither != nullptr && r < n_clips; r++) {
        if (dither[r].kind != R8BGPU_DITHER_OFF && dither[r].kind != R8BGPU_DITHER_TPDF) return fail("unknown dither kind");
        if (dither[r].n_taps != 0)
            return fail("noise-shaped dither is refused: its error feedback runs sequentially through the whole clip");
    }
    for (int r = 0; r < n_clips; r++) {
        if (lens[r] % fi.samples != 0) return fail("lengths of a DSD input must be multiples of 8 samples");
        if (lens[r] > 0 && in.data == nullptr) return fail("null input");
        if (!in.interleaved && (long long) fi.elems(lens[r]) > (long long) in.stride)
            return fail("input stride shorter than clip " + std::to_string(r));
    }
    for (size_t k = 0; k < c.row_len.size(); k++) {
        if (c.row_len[k] > 0 && out.data == nullptr) return fail("null output");
        if (!out.interleaved && c.row_len[k] > (long long) out.stride)
            return fail("output stride shorter than " + c.row_kind() + " " + std::to_string(k));
    }
    if (in.interleaved && in.stride < (size_t) n_clips) return fail("interleaved stride smaller than the clip count");
    if (out.interleaved && out.stride < c.row_len.size()) return fail("interleaved stride smaller than the " + c.row_kind() + " count");
    // (the plans of a mixed batch share one MaxInLen)
    B = b->plan->max_in_len - b->plan->max_in_len % fi.samples;
    if (B <= 0) return fail("MaxInLen holds no whole element of this format");
    return true;
}

// One ordinary batch's share of a checked long-clip call: the spans (whole clips or crops of the caller's clips) laid out
// on its lanes.  Input rows, dither settings and messages of a clip use the caller's index, output rows the span's row;
// everything runs on the batch's stream.  begin() makes the staging (after the clear), then each step() issues one
// ragged call or one flush, so that the parts of a mixed batch can take turns.
struct OneshotJob {
    r8bgpu_batch* b;
    std::string w;
    r8bgpu_buffer in, out;
    FormatElem fi, fo;
    const r8bgpu_dither* dither;
    bool host;
    long long B;
    std::vector<OneshotSpan> spans;
    std::vector<long long> lens, op; // per span: its clip's length and flush target
    OneshotLayout L;
    size_t round = 0, first = 0, last = 0;
    long long call = -1; // -1: the round is not seeded yet; calls[round]: its flush is next
    std::vector<int> seg_of;

    OneshotJob(r8bgpu_batch* b_, const std::string& w_, const r8bgpu_buffer& in_, const r8bgpu_buffer& out_,
               const r8bgpu_dither* dither_, bool host_, long long B_, std::vector<OneshotSpan> spans_, const long long* all_lens,
               const std::vector<long long>& all_op)
        : b(b_), w(w_), in(in_), out(out_), fi(format_elem(in_.format)), fo(format_elem(out_.format)), dither(dither_),
          host(host_), B(B_), spans(std::move(spans_))
    {
        for (const OneshotSpan& s : spans) {
            lens.push_back(all_lens[s.clip]);
            op.push_back(all_op[(size_t) s.clip]);
        }
        oneshot_layout(*b->plan, B, b->n_ch, spans, all_lens, true, L);
    }

    bool fail(const std::string& m) const
    {
        set_err(w + ": " + m);
        return false;
    }
    const unsigned char* clip_in(int r) const
    {
        return (const unsigned char*) in.data + (in.interleaved ? (size_t) r : (size_t) r * in.stride) * fi.bytes;
    }
    unsigned char* row_out(int r) const
    {
        return (unsigned char*) out.data + (out.interleaved ? (size_t) r : (size_t) r * out.stride) * fo.bytes;
    }
    void dith(int r, OneshotRec& q) const
    {
        const bool on = dither != nullptr && dither[r].kind == R8BGPU_DITHER_TPDF && is_int_format(out.format);
        q.dither = on ? 1 : 0;
        q.seed = on ? dither[r].seed : 0;
    }
    bool done() const { return round >= L.calls.size(); }

    bool begin()
    {
        const size_t n_ch = (size_t) b->n_ch;
        if (!ensure_staging(b) || !ensure_ragged_state(b) || (host && !ensure_raw_staging(b, true, true))) return false;
        if (!b->osx) {
            std::unique_ptr<OneshotStaging> x(new OneshotStaging);
            if (!x->rec.create(b->dev_bytes, 2 * n_ch, "oneshot: cudaMalloc(records)", "oneshot: cudaMallocHost(records)",
                               "oneshot: event") ||
                !cuda_ok(cudaEventCreateWithFlags(x->h2d.put(), cudaEventDisableTiming), "oneshot: event"))
                return false;
            b->osx = std::move(x);
        }
        return !host || b->osx->h_in.grow(n_ch * fi.span(B), "oneshot: cudaMallocHost(in)");
    }

    // host form: the scatter writes planar rows of `row_elems` elements into dev_out; the first max_n elements of each
    // row (every lane's kept slice) come back and go to the clips
    struct Pend {
        int r; // the caller's clip
        long long pos, n;
    };
    bool scatter(const std::vector<Pend>& pend, long long max_n, unsigned char* dev_out, size_t row_elems)
    {
        OneshotStaging& ox = *b->osx;
        const int n_ch = b->n_ch;
        const cudaStream_t st = b->stream;
        if (!launch_oneshot_scatter(out.format, host ? false : out.interleaved != 0, host ? 0 : out.stride, out.scale,
                                    ox.rec.d + n_ch, max_n, n_ch, st))
            return false;
        if (!host || max_n <= 0) return true;
        const size_t rb = row_elems * (size_t) fo.bytes, kb = (size_t) max_n * fo.bytes;
        if (!ox.h_out.grow((size_t) n_ch * kb, "oneshot: cudaMallocHost(out)") ||
            !cuda_ok(cudaMemcpy2DAsync(ox.h_out, kb, dev_out, rb, kb, (size_t) n_ch, cudaMemcpyDeviceToHost, st), (w + ": D2H").c_str()) ||
            !cuda_ok(cudaStreamSynchronize(st), (w + ": sync").c_str()))
            return false;
        for (int c = 0; c < n_ch; c++) {
            const Pend& p = pend[(size_t) c];
            if (p.n <= 0) continue;
            const unsigned char* src = ox.h_out + (size_t) c * kb;
            unsigned char* dst = row_out(p.r);
            if (!out.interleaved) memcpy(dst + (size_t) p.pos * fo.bytes, src, (size_t) p.n * fo.bytes);
            else
                for (long long k = 0; k < p.n; k++)
                    memcpy(dst + (size_t) (p.pos + k) * out.stride * fo.bytes, src + (size_t) k * fo.bytes, (size_t) fo.bytes);
        }
        return true;
    }

    // seed: every lane takes its segment's start state (idle lanes: a cleared one) over zeroed rings
    bool seed()
    {
        const Plan& P = *b->plan;
        const int n_ch = b->n_ch;
        const size_t ns = P.stages.size();
        last = first;
        while (last < L.segs.size() && L.segs[last].round == (int) round) last++;
        seg_of.assign((size_t) n_ch, -1);
        for (size_t i = first; i < last; i++) seg_of[(size_t) L.segs[i].lane] = (int) i;
        if (ns == 0) return true;
        std::vector<Schedule> sched((size_t) n_ch);
        std::vector<int> lanes((size_t) n_ch);
        std::vector<StateSeg> zs;
        long long span = 0;
        for (int c = 0; c < n_ch; c++) {
            lanes[(size_t) c] = c;
            Schedule& S = sched[(size_t) c];
            if (seg_of[(size_t) c] >= 0) S = L.start[(size_t) seg_of[(size_t) c]];
            else S.init(&P);
            for (size_t j = 0; j < ns; j++) {
                const StageDev& d = b->dev[j];
                StateSeg z;
                memset(&z, 0, sizeof z);
                z.ring = d.ring + (size_t) c * (size_t) d.ring_cap;
                z.mask = d.ring_cap - 1;
                z.a0 = S.n_in[j]; // an empty window: the whole row becomes zeros
                zs.push_back(z);
                span = std::max(span, d.ring_cap);
            }
        }
        if (!run_segments(b, zs, span, 2, b->stream)) return false;
        b->links_fresh = true;
        channel_schedules(b);
        b->rag.install(lanes.data(), n_ch, sched.data());
        b->diverged = !b->rag.converged();
        if (!b->diverged) b->sched = b->rag.groups[0];
        return true;
    }

    // one block call of the round: every lane of it advances by up to B samples of its segment
    bool block_call()
    {
        const Plan& P = *b->plan;
        OneshotStaging& ox = *b->osx;
        const int n_ch = b->n_ch;
        const size_t ns = P.stages.size(), in_cap = (size_t) P.max_in_len, o_cap = staging_out_cap(P.max_out_len);
        const size_t in_row = fi.span(B), out_row_in = o_cap * (size_t) fo.bytes;
        const cudaStream_t st = b->stream;
        OneshotRec* h = ox.rec.next((w + ": records").c_str());
        if (h == nullptr) return false;
        // h_in still feeds the previous call's upload until that has run
        if (host && !cuda_ok(cudaEventSynchronize(ox.h2d), (w + ": H2D").c_str())) return false;
        std::vector<int> lens_c((size_t) n_ch, 0);
        std::vector<long long> at((size_t) n_ch, 0);
        int max_len = 0;
        for (int c = 0; c < n_ch; c++) {
            OneshotRec& q = h[c];
            memset(&q, 0, sizeof q);
            const int i = seg_of[(size_t) c];
            if (i < 0) continue;
            const r8bgpu_oneshot_seg& s = L.segs[(size_t) i];
            const long long a = s.start + call * B;
            if (a >= s.p1) continue;
            const int n = (int) std::min(B, s.p1 - a);
            lens_c[(size_t) c] = n;
            at[(size_t) c] = a;
            max_len = std::max(max_len, n);
            q.row = b->st_in + (size_t) c * in_cap;
            q.n = n;
            if (host) {
                unsigned char* dst = ox.h_in + (size_t) c * in_row;
                const unsigned char* src = clip_in(spans[(size_t) s.clip].clip);
                const size_t e0 = fi.elems(a), ne = fi.elems(n);
                if (!in.interleaved) memcpy(dst, src + e0 * fi.bytes, ne * fi.bytes);
                else
                    for (size_t k = 0; k < ne; k++)
                        memcpy(dst + k * fi.bytes, src + (e0 + k) * in.stride * fi.bytes, (size_t) fi.bytes);
                q.raw = b->raw_in + (size_t) c * in_row;
                q.pos = 0;
            } else {
                q.raw = clip_in(spans[(size_t) s.clip].clip);
                q.pos = a;
            }
        }
        RaggedSchedule::Step step;
        if (ns > 0) channel_schedules(b).plan_call(lens_c.data(), step);
        // the kept slice of each lane's outputs of this call
        long long max_n = 0;
        std::vector<Pend> pend((size_t) n_ch, Pend{0, 0, 0});
        for (int c = 0; c < n_ch; c++) {
            OneshotRec& q = h[n_ch + c];
            memset(&q, 0, sizeof q);
            const int i = seg_of[(size_t) c];
            if (i < 0) continue;
            const r8bgpu_oneshot_seg& s = L.segs[(size_t) i];
            const OneshotSpan& sp = spans[(size_t) s.clip]; // its output row starts at output sp.e0
            long long o0 = at[(size_t) c], o1 = o0 + lens_c[(size_t) c];
            const double* base = b->st_in + (size_t) c * in_cap;
            if (ns > 0) {
                const StageCall& k = step.calls[(size_t) step.key_of[(size_t) c]][ns - 1];
                o0 = k.e0;
                o1 = k.e1;
                base = b->st_out + (size_t) c * o_cap;
            }
            const long long k0 = std::max(o0, s.e0), k1 = std::min(o1, s.e1);
            if (k1 <= k0) continue;
            q.row = const_cast<double*>(base) + (k0 - o0);
            q.n = k1 - k0;
            q.n0 = k0;
            dith(sp.clip, q);
            q.raw = host ? b->raw_out + (size_t) c * out_row_in : row_out(sp.row);
            q.pos = host ? 0 : k0 - sp.e0;
            pend[(size_t) c] = Pend{sp.row, k0 - sp.e0, k1 - k0};
            max_n = std::max(max_n, q.n);
        }
        if (!ox.rec.upload(0, 2 * (size_t) n_ch, st, (w + ": record upload").c_str())) return false;
        if (host && max_len > 0 &&
            (!cuda_ok(cudaMemcpyAsync(b->raw_in, ox.h_in, (size_t) n_ch * in_row, cudaMemcpyHostToDevice, st), (w + ": H2D").c_str()) ||
             !cuda_ok(cudaEventRecord(ox.h2d, st), (w + ": H2D").c_str())))
            return false;
        if (!launch_oneshot_gather(in.format, host ? false : in.interleaved != 0, host ? 0 : in.stride, in.scale, ox.rec.d,
                                   max_len, n_ch, st))
            return fail("gather: unsupported format");
        if (max_len > 0) b->launches++;
        if (ns > 0) {
            if (!launch_ragged(b, b->rag, step, b->st_in, in_cap, b->st_out, o_cap, st)) return false;
            adopt_step(b, step);
        }
        if (!scatter(pend, max_n, b->raw_out, o_cap)) return false;
        if (max_n > 0) b->launches++;
        return true;
    }

    // the round's flush: the lanes of clips' last segments run to oplens
    bool flush()
    {
        const Plan& P = *b->plan;
        OneshotStaging& ox = *b->osx;
        const int n_ch = b->n_ch;
        const size_t ns = P.stages.size();
        const cudaStream_t st = b->stream;
        std::vector<int> fl;
        std::vector<long long> tg;
        for (size_t i = first; i < last; i++)
            if (L.seg_flush[i]) {
                fl.push_back(L.segs[i].lane);
                tg.push_back(op[(size_t) L.segs[i].clip]);
            }
        FlushJob job;
        std::vector<long long> fbase((size_t) n_ch, 0);
        std::vector<int> fcount((size_t) n_ch, 0);
        double* rows = nullptr;
        size_t rstride = 0;
        if (ns > 0) {
            if (!plan_batch_flush(b, w.c_str(), fl.data(), (int) fl.size(), tg.data(), true, INT_MAX, job)) return false;
            if (!ensure_flush_staging(b, job.max_count + 1, host)) return false;
            if (job.max_count > 0 && !launch_flush(b, job, b->fl_out, b->fl_cap, st)) return false;
            for (int c = 0; c < n_ch; c++) {
                fbase[(size_t) c] = job.out_base[(size_t) c];
                fcount[(size_t) c] = job.counts[(size_t) c];
            }
            rows = b->fl_out;
            rstride = b->fl_cap;
        } else { // passthrough: the tail is silence up to oplens, after the clip's own samples
            long long mx = 0;
            for (size_t i = 0; i < fl.size(); i++) {
                const int c = fl[i];
                fbase[(size_t) c] = lens[(size_t) L.segs[(size_t) seg_of[(size_t) c]].clip];
                fcount[(size_t) c] = (int) std::max(0LL, tg[i] - fbase[(size_t) c]);
                mx = std::max(mx, (long long) fcount[(size_t) c]);
            }
            if (host && !ensure_flush_staging(b, (int) mx + 1, true)) return false;
        }
        OneshotRec* h = ox.rec.next((w + ": records").c_str());
        if (h == nullptr) return false;
        long long max_n = 0;
        std::vector<Pend> pend((size_t) n_ch, Pend{0, 0, 0});
        for (int c = 0; c < n_ch; c++) {
            OneshotRec& q = h[n_ch + c];
            memset(&q, 0, sizeof q);
            const int i = seg_of[(size_t) c];
            if (i < 0 || fcount[(size_t) c] <= 0) continue;
            const r8bgpu_oneshot_seg& s = L.segs[(size_t) i];
            const OneshotSpan& sp = spans[(size_t) s.clip];
            const long long o0 = fbase[(size_t) c], k0 = std::max(o0, s.e0), k1 = std::min(o0 + fcount[(size_t) c], s.e1);
            if (k1 <= k0) continue;
            q.row = rows != nullptr ? rows + (size_t) c * rstride + (k0 - o0) : nullptr;
            q.n = k1 - k0;
            q.n0 = k0;
            dith(sp.clip, q);
            q.raw = host ? b->fl_raw + (size_t) c * b->fl_cap * fo.bytes : row_out(sp.row);
            q.pos = host ? 0 : k0 - sp.e0;
            pend[(size_t) c] = Pend{sp.row, k0 - sp.e0, k1 - k0};
            max_n = std::max(max_n, q.n);
        }
        if (!ox.rec.upload(n_ch, (size_t) n_ch, st, (w + ": record upload").c_str())) return false;
        if (!scatter(pend, max_n, b->fl_raw, b->fl_cap)) return false;
        if (max_n > 0) b->launches++;
        return ns == 0 || finish_flush(b, job, st);
    }

    // Issues the next block call or flush (seeding a round first); false on an error.
    bool step()
    {
        if (call < 0) {
            if (!seed()) return false;
            call = 0;
        }
        if (call < L.calls[round]) {
            if (!block_call()) return false;
            call++;
        } else {
            if (L.flush[round] && !flush()) return false;
            call = L.calls[round] + 1;
        }
        if (call >= L.calls[round] + (L.flush[round] ? 1 : 0)) { // the round is issued
            first = last;
            round++;
            call = -1;
        }
        return true;
    }
};

// The kinds of long-clip entry point, each with its own gate: whole clips on an ordinary batch
// (r8bgpu_batch_oneshot*), whole clips with a plan index each (*_mixed), crops (*_crops*).
enum OneshotEntry { ONESHOT_ORDINARY, ONESHOT_MIXED, ONESHOT_CROPS };

static bool oneshot_gate(const std::string& w, const r8bgpu_batch* b, OneshotEntry e, int n_clips, const int* plan_of_clip)
{
    const char* why = nullptr;
    if (e == ONESHOT_ORDINARY && (b->front || b->mixed)) why = "mixed and multi-device batches are refused: use an ordinary single-device batch";
    else if (e != ONESHOT_ORDINARY && b->front) why = "R8BGPU_DEVICE_ALL batches are refused: use one batch per device";
    else if (e == ONESHOT_MIXED && n_clips > 0 && plan_of_clip == nullptr) why = "null plan_of_clip";
    if (why != nullptr) set_err(w + ": " + why);
    return why == nullptr;
}

// The parts of batch b (a mixed batch's ordinary batches, or b itself) and their plans
static std::vector<r8bgpu_batch*> oneshot_parts(r8bgpu_batch* b, std::vector<const Plan*>& plans)
{
    std::vector<r8bgpu_batch*> parts;
    if (b->mixed)
        for (const auto& pb : b->mixed->parts) parts.push_back(pb.get());
    else
        parts.push_back(b);
    plans.clear();
    for (r8bgpu_batch* pb : parts) plans.push_back(pb->plan);
    return parts;
}

// Runs checked jobs of batch b (one per part of a mixed batch, or one on an ordinary batch): cleared before and after,
// the parts on their own streams after a fork from the batch stream, their calls issued round-robin; the batch stream
// joins them.
static int oneshot_jobs_run(r8bgpu_batch* b, const std::string& w, std::vector<std::unique_ptr<OneshotJob>>& jobs)
{
    DeviceGuard g(b->device);
    if (r8bgpu_batch_clear(b) != 0) return -1;
    for (auto& j : jobs)
        if (!j->begin()) return -1;
    const cudaStream_t st = b->stream;
    if (b->mixed) mixed_fork(b, st);
    bool ok = true, more = true;
    while (ok && more) { // one call per part at a time
        more = false;
        for (size_t k = 0; ok && k < jobs.size(); k++) {
            if (jobs[k]->done()) continue;
            ok = jobs[k]->step();
            more = more || !jobs[k]->done();
        }
    }
    if (b->mixed) mixed_join(b, st);
    if (!ok) return -1;
    if (!cuda_ok(cudaStreamSynchronize(st), (w + ": sync").c_str()) || !cuda_ok(cudaGetLastError(), (w + ": kernel launch").c_str()))
        return -1;
    return r8bgpu_batch_clear(b);
}

// The forward of every long-clip entry point: what = its name; host: in / out are host buffers.  Each part with rows
// runs them as one OneshotJob; a whole-clip call on an ordinary batch makes its staging even when it has no clips.
static int oneshot_run(r8bgpu_batch* b, const char* what, OneshotEntry e, const r8bgpu_buffer* pin, int n_clips,
                       const int* plan_of_clip, const long long* lens, const long long* oplens, int n_crops,
                       const r8bgpu_crop* crops, const r8bgpu_buffer* pout, const r8bgpu_dither* dither, bool host)
{
    const std::string w(what);
    if (b == nullptr || pin == nullptr || pout == nullptr) {
        set_err(w + ": bad arguments");
        return -1;
    }
    std::vector<const Plan*> plans;
    const std::vector<r8bgpu_batch*> parts = oneshot_parts(b, plans);
    OneshotCall c;
    long long B = 0;
    if (!oneshot_gate(w, b, e, n_clips, plan_of_clip) ||
        !oneshot_call(w, w, plans, b->mixed != nullptr, n_clips, plan_of_clip, lens, oplens, e == ONESHOT_CROPS, n_crops, crops, c) ||
        !oneshot_args(w, b, *pin, *pout, c, lens, dither, B))
        return -1;
    std::vector<std::unique_ptr<OneshotJob>> jobs;
    for (size_t p = 0; p < parts.size(); p++)
        if (!c.rows[p].empty() || (!c.cropped && !b->mixed))
            jobs.emplace_back(new OneshotJob(parts[p], w, *pin, *pout, dither, host, B,
                                             oneshot_spans(*plans[p], B, c, p, lens), lens, c.op));
    return oneshot_jobs_run(b, w, jobs);
}

int r8bgpu_batch_oneshot(r8bgpu_batch* b, const r8bgpu_buffer* d_in, int n_clips, const long long* lens, const r8bgpu_buffer* d_out,
                         const long long* oplens, const r8bgpu_dither* dither)
{
    return oneshot_run(b, "batch_oneshot", ONESHOT_ORDINARY, d_in, n_clips, nullptr, lens, oplens, 0, nullptr, d_out, dither, false);
}

int r8bgpu_batch_oneshot_host(r8bgpu_batch* b, const r8bgpu_buffer* h_in, int n_clips, const long long* lens,
                              const r8bgpu_buffer* h_out, const long long* oplens, const r8bgpu_dither* dither)
{
    return oneshot_run(b, "batch_oneshot_host", ONESHOT_ORDINARY, h_in, n_clips, nullptr, lens, oplens, 0, nullptr, h_out, dither, true);
}

int r8bgpu_batch_oneshot_mixed(r8bgpu_batch* b, const r8bgpu_buffer* d_in, int n_clips, const int* plan_of_clip,
                               const long long* lens, const r8bgpu_buffer* d_out, const long long* oplens,
                               const r8bgpu_dither* dither)
{
    return oneshot_run(b, "batch_oneshot_mixed", ONESHOT_MIXED, d_in, n_clips, plan_of_clip, lens, oplens, 0, nullptr, d_out, dither,
                       false);
}

int r8bgpu_batch_oneshot_mixed_host(r8bgpu_batch* b, const r8bgpu_buffer* h_in, int n_clips, const int* plan_of_clip,
                                    const long long* lens, const r8bgpu_buffer* h_out, const long long* oplens,
                                    const r8bgpu_dither* dither)
{
    return oneshot_run(b, "batch_oneshot_mixed_host", ONESHOT_MIXED, h_in, n_clips, plan_of_clip, lens, oplens, 0, nullptr, h_out,
                       dither, true);
}

int r8bgpu_batch_oneshot_crops(r8bgpu_batch* b, const r8bgpu_buffer* d_in, int n_clips, const int* plan_of_clip, const long long* lens,
                               const long long* oplens, int n_crops, const r8bgpu_crop* crops, const r8bgpu_buffer* d_out,
                               const r8bgpu_dither* dither)
{
    return oneshot_run(b, "batch_oneshot_crops", ONESHOT_CROPS, d_in, n_clips, plan_of_clip, lens, oplens, n_crops, crops, d_out,
                       dither, false);
}

int r8bgpu_batch_oneshot_crops_host(r8bgpu_batch* b, const r8bgpu_buffer* h_in, int n_clips, const int* plan_of_clip,
                                    const long long* lens, const long long* oplens, int n_crops, const r8bgpu_crop* crops,
                                    const r8bgpu_buffer* h_out, const r8bgpu_dither* dither)
{
    return oneshot_run(b, "batch_oneshot_crops_host", ONESHOT_CROPS, h_in, n_clips, plan_of_clip, lens, oplens, n_crops, crops, h_out,
                       dither, true);
}

} // extern "C"

// ---- gradients through long clips (r8bgpu_batch_oneshot_adjoint) -----------------------------------------------------
// The twin of a clip (include/r8bgpu.h, "long clips") walked on the host: per stage, the window of gradient samples of its
// output ([g0, ng)) and of its input ([lo, ext): ext is one past the largest input index a kept output reads, lo the
// smallest), and the order-2 interpolator's per-call timing records.  Whole clips keep [0, oplen) with every origin 0;
// a crop keeps [o0, o1).  out0: the first kept output; b0 / nb: a block-exact stage's blocks.
struct AdjGeom {
    std::vector<long long> ng, ext, nb, g0, lo, b0;
    std::vector<std::vector<AdjPolyRec>> rec;
    long long out0 = 0;
};

// Block-exact BlockConv stage s: blocks of il tile-stream samples, windows of M from b * il - prev (the forward tile
// geometry of blockconv_call_fields, whose windows start at m0 - lg).
static void adj_block_geom(const StageDesc& s, int& M, int& il, int& prev)
{
    const BcTile t = blockconv_tile(s, true);
    M = 1 << t.fft_log2;
    il = s.ref_input_len;
    prev = t.lg + s.lp.half_len;
}

// The twin's order-2 timing records of every stage: the walk of a clip of len samples and its flush to oplen
static const char* adjoint_records(const Plan& P, long long len, long long oplen, std::vector<std::vector<AdjPolyRec>>& rec)
{
    const size_t ns = P.stages.size();
    rec.assign(ns, std::vector<AdjPolyRec>());
    if (ns == 0) return nullptr;
    auto take = [&](const std::vector<StageCall>& cs) {
        for (size_t j = 0; j < ns && j < cs.size(); j++) {
            const StageCall& c = cs[j];
            if (P.stages[j].kind != ST_FRAC_POLY || c.e1 <= c.e0) continue;
            AdjPolyRec r;
            r.e0 = c.e0;
            r.p0 = c.p0;
            r.in_pos_shift = c.in_pos_shift;
            r.fpos0 = c.fpos0;
            r.ssr = c.ssr;
            r.dsr = c.dsr;
            r.in_counter0 = c.in_counter0;
            r.in_pos_int0 = c.in_pos_int0;
            rec[j].push_back(r);
        }
    };
    Schedule s;
    s.init(&P);
    std::vector<StageCall> calls;
    const long long B = P.max_in_len;
    for (long long pos = 0; pos < len; pos += B) {
        s.advance((int) std::min(B, len - pos), calls);
        take(calls);
    }
    if (oplen > s.outputs()) {
        if (oplen - s.outputs() > INT_MAX) return "the output past the clip's last input sample exceeds 2^31 - 1 samples";
        FlushPlan f;
        plan_flush(s, oplen, f, true);
        for (const std::vector<StageCall>& c : f.calls) take(c);
    }
    return nullptr;
}

static long long ceil_div_ll(long long a, long long b) { return a >= 0 ? (a + b - 1) / b : -((-a) / b); }

// The windows of outputs [q0, q1) through the chain, from the twin's records.  window false (whole clips): q0 = 0 and
// every origin 0, the extents alone as before.
static const char* adjoint_windows(const Plan& P, std::vector<std::vector<AdjPolyRec>> rec, long long q0, long long q1,
                                   bool window, AdjGeom& g)
{
    const size_t ns = P.stages.size();
    g.ng.assign(ns, 0);
    g.ext.assign(ns, 0);
    g.nb.assign(ns, 0);
    g.g0.assign(ns, 0);
    g.lo.assign(ns, 0);
    g.b0.assign(ns, 0);
    g.rec = std::move(rec);
    g.out0 = window ? q0 : 0;
    long long Q = q1, Qlo = g.out0;
    for (size_t jj = ns; jj-- > 0;) {
        const StageDesc& st = P.stages[jj];
        g.ng[jj] = Q;
        g.g0[jj] = Qlo;
        long long R = 0, lo = 0;
        if (Q > Qlo) {
            switch (st.kind) {
            case ST_BLOCKCONV:
                if (st.block_exact) {
                    int M, il, prev;
                    adj_block_geom(st, M, il, prev);
                    const long long bl = (st.down * (Q - 1) + st.lp.half_len) / il;
                    g.nb[jj] = bl + 1;
                    R = ((bl + 1) * il - 1) / st.up + 1;
                    if (window) { // the window of the first block that holds a kept output
                        g.b0[jj] = (st.down * Qlo + st.lp.half_len) / il;
                        lo = ceil_div_ll(g.b0[jj] * il - prev, st.up);
                    }
                } else {
                    R = (st.down * (Q - 1) + st.lp.half_len) / st.up + 1;
                    lo = ceil_div_ll(st.down * Qlo - st.lp.half_len, st.up);
                }
                break;
            case ST_FRAC_WHOLE:
                R = (Q - 1) * st.in_step / st.out_step + st.bank.filter_len / 2 + 1;
                lo = Qlo * st.in_step / st.out_step - (st.bank.filter_len / 2 - 1);
                break;
            case ST_FRAC_POLY: {
                const std::vector<AdjPolyRec>& rs = g.rec[jj];
                // output j reads [p_j - fll, p_j - fll + flen)
                auto pos = [&](long long j, long long& p) -> bool {
                    size_t k = 0;
                    while (k + 1 < rs.size() && rs[k + 1].e0 <= j) k++;
                    if (rs.empty() || rs[k].e0 > j) return false;
                    const AdjPolyRec& c = rs[k];
                    p = c.p0;
                    if (j > c.e0) {
                        const double np = ((double) (c.in_counter0 + (int) (j - c.e0)) + c.in_pos_shift) * c.ssr / c.dsr;
                        p = c.p0 + ((int) np - c.in_pos_int0);
                    }
                    return true;
                };
                long long p = 0;
                if (!pos(Q - 1, p)) return "no interpolator timing record covers the clip's outputs";
                R = p + st.bank.filter_len / 2 + 1;
                if (window) {
                    if (!pos(Qlo, p)) return "no interpolator timing record covers the clip's outputs";
                    lo = p - (st.bank.filter_len / 2 - 1);
                }
                break;
            }
            case ST_HBUP: { // output 2n reads x[n], output 2n + 1 reads x[n - T + 1 .. n + T]
                const long long e = (Q - 1) & 1 ? Q - 2 : Q - 1, o = (Q - 1) & 1 ? Q - 1 : Q - 2;
                R = e / 2 + 1;
                if (o >= 1) R = std::max(R, (o - 1) / 2 + st.hb_taps + 1);
                lo = (Qlo >> 1) - st.hb_taps + 1;
                break;
            }
            case ST_HBDOWN: // output m reads [2m - 2T + 1, 2m + 2T - 1]; the window starts even (k_hbup writes pairs)
                R = 2 * (Q - 1) + 2 * st.hb_taps;
                lo = 2 * (Qlo - st.hb_taps);
                break;
            }
        }
        g.ext[jj] = std::max(0LL, R);
        g.lo[jj] = window ? std::min(std::max(0LL, lo), g.ext[jj]) : 0;
        if (window && g.ext[jj] <= g.lo[jj]) g.ext[jj] = g.lo[jj] = 0;
        Q = g.ext[jj];
        Qlo = g.lo[jj];
    }
    return nullptr;
}

static const char* adjoint_geometry(const Plan& P, long long len, long long oplen, AdjGeom& g)
{
    std::vector<std::vector<AdjPolyRec>> rec;
    if (const char* why = adjoint_records(P, len, oplen, rec)) return why;
    return adjoint_windows(P, std::move(rec), 0, oplen, false, g);
}

// The call's device scratch: two ping-pong planar fp64 buffers of n_clips rows of `stride` doubles, and for block-exact
// stages the per-block contributions; out: the sizes.
struct AdjScratch {
    long long stride = 0, c_stride = 0, max_nb = 0;
    int n_recs = 0;
    unsigned long long bytes = 0;
};

// Rows are as wide as the widest window: lens / op are each row's input and output ends, x0 its input's first sample.
static AdjScratch adjoint_scratch(const Plan& P, const std::vector<AdjGeom>& G, const long long* lens, const long long* op,
                                  const long long* x0)
{
    AdjScratch a;
    const size_t n = G.size(), ns = P.stages.size();
    for (size_t r = 0; r < n; r++) {
        a.stride = std::max(a.stride, std::max(lens[r] - x0[r], op[r] - G[r].out0));
        for (size_t j = 0; j < ns; j++) {
            a.stride = std::max(a.stride, std::max(G[r].ng[j] - G[r].g0[j], G[r].ext[j] - G[r].lo[j]));
            a.max_nb = std::max(a.max_nb, G[r].nb[j] - G[r].b0[j]);
            a.n_recs = std::max(a.n_recs, (int) G[r].rec[j].size());
        }
    }
    a.stride += 2; // k_hbup writes output pairs
    for (size_t j = 0; j < ns; j++)
        if (P.stages[j].kind == ST_BLOCKCONV && P.stages[j].block_exact) {
            int M, il, prev;
            adj_block_geom(P.stages[j], M, il, prev);
            long long nb = 0;
            for (size_t r = 0; r < n; r++) nb = std::max(nb, G[r].nb[j] - G[r].b0[j]);
            a.c_stride = std::max(a.c_stride, nb * M);
        }
    a.bytes = (unsigned long long) n * (2ULL * (unsigned long long) a.stride + (unsigned long long) a.c_stride) * sizeof(double) +
              (unsigned long long) n * ((unsigned long long) a.n_recs * sizeof(AdjPolyRec) + sizeof(AdjClip) + 2 * sizeof(MapRec));
    return a;
}

// kappa[d] = sum_k nat[k] e^(2 pi i k d / M) (long double radix-2 transform) and the slot order of the forward spectrum
static std::vector<double> adj_kappa(const std::vector<double2>& nat)
{
    const size_t M = nat.size();
    std::vector<long double> re(M), im(M);
    for (size_t k = 0; k < M; k++) {
        re[k] = nat[k].x;
        im[k] = nat[k].y;
    }
    for (size_t i = 1, j = 0; i < M; i++) {
        size_t bit = M >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) {
            std::swap(re[i], re[j]);
            std::swap(im[i], im[j]);
        }
    }
    const long double two_pi = 6.283185307179586476925286766559005768L;
    for (size_t len = 2; len <= M; len <<= 1)
        for (size_t i = 0; i < M; i += len)
            for (size_t k = 0; k < len / 2; k++) {
                const long double a = two_pi * (long double) k / (long double) len, c = cosl(a), s = sinl(a);
                const size_t u = i + k, v = u + len / 2;
                const long double tr = re[v] * c - im[v] * s, ti = re[v] * s + im[v] * c;
                re[v] = re[u] - tr;
                im[v] = im[u] - ti;
                re[u] += tr;
                im[u] += ti;
            }
    std::vector<double> out(M);
    for (size_t d = 0; d < M; d++) out[d] = (double) re[d];
    return out;
}

template <int M>
static void adj_nat_small(const std::vector<double2>& slots, std::vector<double2>& nat)
{
    nat.resize((size_t) M);
    for (int k = 0; k < M; k++) nat[(size_t) k] = slots[(size_t) slot_of<M>(k)];
}

// The block-exact stage's kernel in exact arithmetic: kappa, u and the Nyquist gain (k_blockconv / k_bcl with trunc).
static void adj_block_tables(const StageDesc& s, std::vector<double>& kappa, std::vector<double>& u, double& nyq)
{
    const BcTile t = blockconv_tile(s, true);
    const int M = 1 << t.fft_log2;
    std::vector<double2> slots, tw, tw_m, nat;
    nyq = 0.0;
    if (t.large) {
        build_spectrum_large(s, t.fft_log2, slots, tw, tw_m, &nyq);
        nat.resize((size_t) M);
        for (int k = 0; k < M; k++) nat[(size_t) k] = slots[(size_t) bcl::slot_of_large(k, M / bcl::SUB)];
    } else {
        build_spectrum(s, t.fft_log2, slots, tw, &nyq);
        switch (t.fft_log2) {
        case 6: adj_nat_small<64>(slots, nat); break;
        case 7: adj_nat_small<128>(slots, nat); break;
        case 8: adj_nat_small<256>(slots, nat); break;
        case 9: adj_nat_small<512>(slots, nat); break;
        case 10: adj_nat_small<1024>(slots, nat); break;
        case 11: adj_nat_small<2048>(slots, nat); break;
        case 13: adj_nat_small<8192>(slots, nat); break;
        default: adj_nat_small<4096>(slots, nat); break;
        }
    }
    nat[(size_t) (M / (2 * s.down))] = make_double2(0.0, 0.0); // the forward puts the Nyquist term in this bin instead
    kappa = adj_kappa(nat);
    u.resize((size_t) M);
    const long double pi = 3.141592653589793238462643383279502884L;
    for (int m = 0; m < M; m++) {
        const long double a = pi * (long double) m / (long double) s.down;
        u[(size_t) m] = (double) (cosl(a) + sinl(a));
    }
}

long long r8bgpu_plan_oneshot_adjoint_extents(const r8bgpu_plan* plan, long long len, long long oplen, long long* ext, int cap)
{
    const char* what = "plan_oneshot_adjoint_extents";
    if (plan == nullptr || len < 0 || oplen < 0 || (cap > 0 && ext == nullptr)) {
        set_err(std::string(what) + ": bad arguments");
        return -1;
    }
    const Plan& P = plan->p;
    if (const char* why = oneshot_plan_refusal(P)) {
        set_err(std::string(what) + ": " + why);
        return -1;
    }
    AdjGeom g;
    if (const char* why = adjoint_geometry(P, len, oplen, g)) {
        set_err(std::string(what) + ": " + why);
        return -1;
    }
    for (int j = 0; j < cap && j < (int) g.ext.size(); j++) ext[j] = g.ext[(size_t) j];
    return (long long) g.ext.size();
}

long long r8bgpu_plan_oneshot_adjoint_bytes(const r8bgpu_plan* plan, int n_clips, const long long* lens, const long long* oplens)
{
    const char* what = "plan_oneshot_adjoint_bytes";
    if (plan == nullptr) {
        set_err(std::string(what) + ": bad arguments");
        return -1;
    }
    const Plan& P = plan->p;
    OneshotCall c;
    if (!oneshot_call(what, what, {&P}, false, n_clips, nullptr, lens, oplens, false, 0, nullptr, c)) return -1;
    std::vector<AdjGeom> G((size_t) n_clips);
    for (int r = 0; r < n_clips; r++)
        if (const char* why = adjoint_geometry(P, lens[r], c.op[(size_t) r], G[(size_t) r])) {
            set_err(std::string(what) + ": " + why);
            return -1;
        }
    return (long long) adjoint_scratch(P, G, lens, c.op.data(), std::vector<long long>((size_t) n_clips, 0).data()).bytes;
}

// The gradient buffers of a checked long-clip call: go holds its rows, gi its clips.
static bool adjoint_args(const std::string& w, const r8bgpu_batch* b, const r8bgpu_buffer& go, const r8bgpu_buffer& gi,
                         const OneshotCall& c, const long long* lens)
{
    auto fail = [&](const std::string& m) {
        set_err(w + ": " + m);
        return false;
    };
    const int n_clips = (int) c.plan.size();
    if (dsd_on(b)) return fail("DSD output is on: its modulators run sequentially through a whole clip");
    for (const r8bgpu_buffer* x : {&go, &gi})
        if (x->format != R8BGPU_F64 && x->format != R8BGPU_F32) return fail("gradients are R8BGPU_F64 or R8BGPU_F32 buffers");
    if (go.scale != 1.0 || gi.scale != 1.0) return fail("gradient buffers take scale 1");
    for (int r = 0; r < n_clips; r++) {
        if (lens[r] > 0 && gi.data == nullptr) return fail("null input gradient");
        if (!gi.interleaved && lens[r] > (long long) gi.stride) return fail("input gradient stride shorter than clip " + std::to_string(r));
    }
    for (size_t k = 0; k < c.row_len.size(); k++) {
        if (c.row_len[k] > 0 && go.data == nullptr) return fail("null output gradient");
        if (!go.interleaved && c.row_len[k] > (long long) go.stride)
            return fail("output gradient stride shorter than " + c.row_kind() + " " + std::to_string(k));
    }
    if (go.interleaved && go.stride < c.row_len.size()) return fail("interleaved stride smaller than the " + c.row_kind() + " count");
    if (gi.interleaved && gi.stride < (size_t) n_clips) return fail("interleaved stride smaller than the clip count");
    return true;
}

// One part's share of a checked adjoint call: its rows idx (the caller's indices, ascending) of plan P, whose transposed
// chain runs on the part's stream (the part counts the launches).  The chain's rows are the job's own; the two mapped
// conversions span all n_all caller rows, with extent 0 on the rows of other parts.  prepare() walks the twins (its
// refusals change nothing), alloc() takes the scratch on st, issue() queues the chain and then the frees on st; nothing
// synchronises.  Rows that are crops (r8bgpu_batch_oneshot_crops_adjoint) run their chains over their windows only, and
// k_crop_accum sums each clip's crop rows into its caller row.
struct AdjJob {
    r8bgpu_batch* b;
    const Plan& P;
    cudaStream_t st;
    std::string w;
    std::vector<int> idx;
    int n_all;
    const r8bgpu_crop* crops;         // null: the rows are whole clips
    std::vector<int> clip;            // per row of the job: its clip
    std::vector<long long> lens, op;  // per row of the job: its input's and output's ends
    std::vector<long long> x0;        // per row of the job: its input window's first sample (whole clips: 0)
    std::vector<AdjGeom> G;
    AdjScratch A;
    long long max_op = 0, max_len = 0;
    std::vector<void*> held;
    void* scratch = nullptr;
    MapRec* d_map = nullptr; // [2][n_all]

    AdjJob(r8bgpu_batch* part, const std::string& w_, const OneshotCall& c, size_t p, const long long* all_lens)
        : b(part), P(*part->plan), st(part->stream), w(w_), idx(c.rows[p]), n_all((int) c.row_len.size()),
          crops(c.cropped ? c.crops : nullptr)
    {
        for (int r : idx) {
            clip.push_back(crops != nullptr ? crops[r].clip : r);
            lens.push_back(all_lens[clip.back()]);
            op.push_back(c.op[(size_t) clip.back()]);
        }
    }
    ~AdjJob() { release(); }

    bool fail(const std::string& m) const
    {
        set_err(w + ": " + m);
        return false;
    }
    // one twin walk per clip; each row's windows from its clip's records
    bool prepare()
    {
        const size_t n = idx.size();
        G.assign(n, AdjGeom());
        x0.assign(n, 0);
        std::map<int, std::vector<std::vector<AdjPolyRec>>> recs;
        for (size_t r = 0; r < n; r++) {
            auto it = recs.find(clip[r]);
            if (it == recs.end()) {
                std::vector<std::vector<AdjPolyRec>> rc;
                if (const char* why = adjoint_records(P, lens[r], op[r], rc)) return fail(why);
                it = recs.emplace(clip[r], std::move(rc)).first;
            }
            const long long o0 = crops != nullptr ? crops[idx[r]].o0 : 0, o1 = crops != nullptr ? crops[idx[r]].o1 : op[r];
            if (const char* why = adjoint_windows(P, it->second, o0, o1, crops != nullptr, G[r])) return fail(why);
            if (crops != nullptr) { // the crop's input window
                const bool ns0 = P.stages.empty();
                const long long hi = std::min(lens[r], ns0 ? o1 : G[r].ext[0]), lo = ns0 ? o0 : G[r].lo[0];
                x0[r] = hi > lo ? lo : 0; // an empty window is [0, 0): k_hbup's pairs start even
                lens[r] = hi > lo ? hi : 0;
                op[r] = o1;
            }
        }
        A = adjoint_scratch(P, G, lens.data(), op.data(), x0.data());
        for (size_t r = 0; r < n; r++) {
            max_op = std::max(max_op, op[r] - G[r].out0);
            max_len = std::max(max_len, lens[r] - x0[r]);
        }
        return true;
    }
    bool dalloc(size_t bytes, void** p)
    {
        *p = nullptr;
        if (cudaMallocAsync(p, std::max<size_t>(bytes, 16), st) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        held.push_back(*p);
        return true;
    }
    // queued on st, after whatever uses the memory
    void release()
    {
        for (void* p : held) cudaFreeAsync(p, st);
        held.clear();
    }
    bool alloc()
    {
        if (!dalloc((size_t) A.bytes, &scratch)) return fail("cannot allocate " + std::to_string(A.bytes) + " bytes of scratch on the device");
        const size_t n = idx.size();
        if ((size_t) n_all == n) { // every caller row: the scratch's own records
            d_map = (MapRec*) ((AdjClip*) ((AdjPolyRec*) ((double*) scratch + n * (2 * (size_t) A.stride + (size_t) A.c_stride)) +
                                          n * (size_t) A.n_recs) + n);
            return true;
        }
        void* m = nullptr;
        if (!dalloc(2 * (size_t) n_all * sizeof(MapRec), &m)) return fail("cannot allocate the conversion records on the device");
        d_map = (MapRec*) m;
        return true;
    }

    bool issue(const r8bgpu_buffer& go, const r8bgpu_buffer& gi)
    {
        const size_t n = idx.size();
        const int nl = (int) n;
        double* buf[2] = {(double*) scratch, (double*) scratch + n * (size_t) A.stride};
        double* contrib = buf[1] + n * (size_t) A.stride;
        AdjPolyRec* d_rec = (AdjPolyRec*) (contrib + n * (size_t) A.c_stride);
        AdjClip* d_clip = (AdjClip*) (d_rec + n * (size_t) A.n_recs);
        auto up = [&](void* dst, const void* src, size_t bytes) {
            return bytes == 0 || cuda_ok(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st), (w + ": upload").c_str());
        };
        auto table = [&](const void* src, size_t bytes, const void** out) {
            void* p = nullptr;
            if (!dalloc(bytes, &p)) return fail("cannot allocate " + std::to_string(bytes) + " bytes for a stage table");
            *out = p;
            return up(p, src, bytes);
        };
        bool ok = cuda_ok(cudaMemsetAsync(scratch, 0, 2 * n * (size_t) A.stride * sizeof(double), st), (w + ": memset").c_str());
        // the output gradient, widened into buf[0]: the group's caller rows to its scratch rows
        std::vector<MapRec> map((size_t) n_all, MapRec{nullptr, 0});
        for (size_t r = 0; r < n; r++) map[(size_t) idx[r]] = MapRec{buf[0] + r * (size_t) A.stride, op[r] - G[r].out0};
        // the mapped conversions take the channel from gridDim.y: clips go in groups of at most 65535
        auto convert = [&](bool to_f64, const r8bgpu_buffer& buf_, const MapRec* rec, long long cnt) {
            for (int c0 = 0; c0 < n_all; c0 += 65535) {
                const int nc = std::min(n_all - c0, 65535);
                unsigned char* raw = (unsigned char*) buf_.data +
                                     (buf_.interleaved ? (size_t) c0 : (size_t) c0 * buf_.stride) * (size_t) format_bytes(buf_.format);
                const bool k = to_f64 ? launch_to_f64_mapped(buf_.format, raw, buf_.interleaved != 0, buf_.stride, rec + c0, (int) cnt, nc, 1.0, st)
                                      : launch_from_f64_mapped(buf_.format, raw, buf_.interleaved != 0, buf_.stride, rec + c0, (int) cnt, nc, 1.0, st);
                if (!k) return false;
                b->launches++;
            }
            return true;
        };
        ok = ok && up(d_map, map.data(), (size_t) n_all * sizeof(MapRec)) && convert(true, go, d_map, max_op);
        const size_t ns = P.stages.size();
        int cur = 0;
        for (size_t jj = ns; ok && jj-- > 0;) {
            const StageDesc& s = P.stages[jj];
            std::vector<AdjClip> cl(n);
            std::vector<AdjPolyRec> recs;
            long long max_nx = 0, max_nb = 0;
            for (size_t r = 0; r < n; r++) {
                AdjClip& c = cl[r];
                c.ng = G[r].ng[jj];
                c.nx = jj == 0 ? lens[r] : G[r].ext[jj];
                c.nb = G[r].nb[jj];
                c.rec0 = (int) recs.size();
                c.nrec = (int) G[r].rec[jj].size();
                c.g0 = G[r].g0[jj];
                c.x0 = jj == 0 ? x0[r] : G[r].lo[jj];
                c.b0 = G[r].b0[jj];
                recs.insert(recs.end(), G[r].rec[jj].begin(), G[r].rec[jj].end());
                max_nx = std::max(max_nx, c.nx - c.x0);
                max_nb = std::max(max_nb, c.nb - c.b0);
            }
            AdjParams p;
            memset(&p, 0, sizeof p);
            p.g = buf[cur];
            p.g_stride = A.stride;
            p.x = buf[cur ^ 1];
            p.x_stride = A.stride;
            p.clip = d_clip;
            ok = ok && up(d_clip, cl.data(), n * sizeof(AdjClip)) && up(d_rec, recs.data(), recs.size() * sizeof(AdjPolyRec));
            if (!ok) break;
            p.rec = d_rec;
            const void* t0 = nullptr;
            const void* t1 = nullptr;
            switch (s.kind) {
            case ST_BLOCKCONV:
                p.L = s.lp.half_len;
                p.U = s.up;
                p.D = s.down;
                if (!s.block_exact) {
                    ok = table(s.lp.taps.data(), s.lp.taps.size() * sizeof(double), &t0);
                    p.h = (const double*) t0;
                    if (ok) launch_bc_adj(p, max_nx, nl, st);
                } else {
                    std::vector<double> kappa, u;
                    adj_block_tables(s, kappa, u, p.nyq);
                    adj_block_geom(s, p.M, p.il, p.prev);
                    ok = table(kappa.data(), kappa.size() * sizeof(double), &t0) && table(u.data(), u.size() * sizeof(double), &t1);
                    p.kappa = (const double*) t0;
                    p.u = (const double*) t1;
                    p.contrib = contrib;
                    p.c_stride = A.c_stride;
                    if (ok) launch_bcx_adj(p, max_nb, max_nx, nl, st);
                    b->launches++;
                }
                b->launches++;
                break;
            case ST_FRAC_WHOLE:
            case ST_FRAC_POLY:
                ok = table(s.bank.table.data(), s.bank.table.size() * sizeof(double), &t0);
                p.bank = (const double*) t0;
                p.flen = s.bank.filter_len;
                p.fll = s.bank.filter_len / 2 - 1;
                p.in_step = s.in_step;
                p.out_step = s.out_step;
                p.fracs = s.bank.fracs;
                if (ok) launch_frac_adj(p, s.kind == ST_FRAC_POLY, max_nx, nl, st);
                b->launches++;
                break;
            case ST_HBUP:
            case ST_HBDOWN: {
                // the transpose of a half-band stage is the other direction's stage with the same taps (DESIGN.md K9)
                std::vector<RaggedRec> rr(n);
                for (size_t r = 0; r < n; r++) { // the windows: x from x0 (even for k_hbup's pairs), g from g0
                    memset(&rr[r], 0, sizeof(RaggedRec));
                    rr[r].e0 = cl[r].x0;
                    rr[r].e1 = cl[r].nx;
                    rr[r].dst_base = cl[r].x0;
                    rr[r].cur_base = cl[r].g0;
                    rr[r].avail = cl[r].ng;
                }
                const void* d_rr = nullptr;
                static const double zeros[64] = {0};
                const void* d_zero = nullptr;
                ok = table(rr.data(), n * sizeof(RaggedRec), &d_rr) && table(zeros, sizeof zeros, &d_zero);
                if (!ok) break;
                HbParams hp;
                memset(&hp, 0, sizeof hp);
                hp.ntaps = s.hb_taps;
                hp.e0 = 0;
                hp.e1 = max_nx + (max_nx & 1); // k_hbup's grid: a pair for every output of an odd row too
                for (int k = 0; k < s.hb_taps; k++) hp.taps[k] = s.hb[(size_t) k];
                SrcView sv;
                memset(&sv, 0, sizeof sv);
                sv.ring = (const double*) d_zero;
                sv.ring_stride = 0;
                sv.ring_mask = 63;
                sv.cur = p.g;
                sv.cur_stride = A.stride;
                sv.cur_base = 0;
                sv.avail = LLONG_MAX;
                sv.cur_scale = 1.0;
                DstView dv;
                memset(&dv, 0, sizeof dv);
                dv.ptr = p.x;
                dv.stride = A.stride;
                dv.mask = -1;
                dv.scale = 1.0;
                // these kernels take the channel from gridDim.y: clips go in groups of at most 65535
                for (int c0 = 0; c0 < nl; c0 += 65535) {
                    const int nc = std::min(nl - c0, 65535);
                    SrcView svc = sv;
                    DstView dvc = dv;
                    svc.cur += (size_t) c0 * (size_t) A.stride;
                    dvc.ptr += (size_t) c0 * (size_t) A.stride;
                    const RaggedRec* rrc = (const RaggedRec*) d_rr + c0;
                    if (s.kind == ST_HBUP) launch_hbdown(hp, svc, dvc, nc, st, rrc);
                    else launch_hbup(hp, svc, dvc, nc, st, rrc);
                    b->launches++;
                }
                break;
            }
            }
            ok = ok && cuda_ok(cudaGetLastError(), (w + ": kernel launch").c_str());
            cur ^= 1;
        }
        // the input gradient: buf[cur] rows narrowed into the group's caller rows, lens[r] samples each (a passthrough
        // plan's rows are the output gradient, zero past oplens); crops: each clip's crop rows summed over their hull
        if (ok && crops != nullptr) {
            std::map<int, std::vector<size_t>> by_clip; // rows in ascending crop order
            for (size_t r = 0; r < n; r++)
                if (lens[r] > x0[r]) by_clip[clip[r]].push_back(r);
            std::vector<CropAccRow> rows;
            std::vector<CropAccClip> cc;
            long long max_hull = 0;
            for (const auto& kv : by_clip) {
                CropAccClip c;
                c.lo = LLONG_MAX;
                c.hi = 0;
                c.k0 = (int) rows.size();
                c.nk = (int) kv.second.size();
                c.out = kv.first;
                for (size_t r : kv.second) {
                    rows.push_back(CropAccRow{x0[r], lens[r], (long long) r});
                    c.lo = std::min(c.lo, x0[r]);
                    c.hi = std::max(c.hi, lens[r]);
                }
                max_hull = std::max(max_hull, c.hi - c.lo);
                cc.push_back(c);
            }
            const void* d_rows = nullptr;
            const void* d_cc = nullptr;
            ok = table(rows.data(), rows.size() * sizeof(CropAccRow), &d_rows) && table(cc.data(), cc.size() * sizeof(CropAccClip), &d_cc);
            if (ok && !cc.empty()) {
                CropAccParams q;
                q.x = buf[cur];
                q.x_stride = A.stride;
                q.rows = (const CropAccRow*) d_rows;
                q.clips = (const CropAccClip*) d_cc;
                q.out = gi.data;
                q.fmt = gi.format == R8BGPU_F64 ? FMT_F64 : FMT_F32;
                q.interleaved = gi.interleaved != 0;
                q.out_stride = (long long) gi.stride;
                launch_crop_accum(q, max_hull, (int) cc.size(), st);
                b->launches++;
                ok = cuda_ok(cudaGetLastError(), (w + ": kernel launch").c_str());
            }
        } else if (ok) {
            for (size_t r = 0; r < n; r++) map[(size_t) idx[r]] = MapRec{buf[cur] + r * (size_t) A.stride, lens[r]};
            ok = up(d_map + n_all, map.data(), (size_t) n_all * sizeof(MapRec));
            ok = ok && convert(false, gi, d_map + n_all, max_len);
        }
        release();
        return ok;
    }
};

// The adjoint of a checked call whose groups are prepared: one AdjJob per group of clips, each on its stream (a mixed
// batch: its part's, forked from the batch stream and joined to it; an ordinary batch: the batch stream).  Every group is
// allocated before any runs, and the call finishes before it returns.
static int adjoint_run(r8bgpu_batch* b, const std::string& w, std::vector<std::unique_ptr<AdjJob>>& jobs,
                       const r8bgpu_buffer& go, const r8bgpu_buffer& gi)
{
    for (auto& j : jobs)
        if (j->max_op > INT_MAX || j->max_len > INT_MAX) {
            set_err(w + ": clips and outputs are limited to 2^31 - 1 samples");
            return -1;
        }
    DeviceGuard guard(b->device);
    const cudaStream_t st = b->stream;
    auto finish = [&]() {
        for (auto& j : jobs) j->release();
        if (b->mixed) mixed_join(b, st);
        return cudaStreamSynchronize(st);
    };
    for (auto& j : jobs)
        if (!j->alloc()) {
            const std::string e = r8bgpu_last_error();
            finish();
            set_err(e);
            return -1;
        }
    if (b->mixed) mixed_fork(b, st);
    bool ok = true;
    for (auto& j : jobs) ok = ok && j->issue(go, gi);
    const cudaError_t e = finish();
    if (!ok) return -1;
    if (!cuda_ok(e, (w + ": sync").c_str()) || !cuda_ok(cudaGetLastError(), (w + ": kernel").c_str())) return -1;
    return 0;
}

// The adjoint of every long-clip entry point: one AdjJob per part with rows, run by adjoint_run once every job is
// prepared.
static int adjoint_drive(r8bgpu_batch* b, const char* what, OneshotEntry e, const r8bgpu_buffer* pgo, int n_clips,
                         const int* plan_of_clip, const long long* lens, const long long* oplens, int n_crops,
                         const r8bgpu_crop* crops, const r8bgpu_buffer* pgi)
{
    const std::string wg(what);
    if (b == nullptr || pgo == nullptr || pgi == nullptr) {
        set_err(wg + ": bad arguments");
        return -1;
    }
    // on an ordinary batch the mixed entry answers as r8bgpu_batch_oneshot_adjoint past its gate and plan indices
    const std::string w = e == ONESHOT_MIXED && !b->mixed ? "batch_oneshot_adjoint" : wg;
    std::vector<const Plan*> plans;
    const std::vector<r8bgpu_batch*> parts = oneshot_parts(b, plans);
    OneshotCall c;
    if (!oneshot_gate(wg, b, e, n_clips, plan_of_clip) ||
        !oneshot_call(w, wg, plans, b->mixed != nullptr, n_clips, plan_of_clip, lens, oplens, e == ONESHOT_CROPS, n_crops, crops, c) ||
        !adjoint_args(w, b, *pgo, *pgi, c, lens))
        return -1;
    std::vector<std::unique_ptr<AdjJob>> jobs;
    for (size_t p = 0; p < parts.size(); p++)
        if (!c.rows[p].empty()) jobs.emplace_back(new AdjJob(parts[p], w, c, p, lens));
    for (auto& j : jobs)
        if (!j->prepare()) return -1;
    if (jobs.empty()) return 0;
    return adjoint_run(b, w, jobs, *pgo, *pgi);
}

int r8bgpu_batch_oneshot_adjoint(r8bgpu_batch* b, const r8bgpu_buffer* d_gout, int n_clips, const long long* lens,
                                 const long long* oplens, const r8bgpu_buffer* d_gin)
{
    return adjoint_drive(b, "batch_oneshot_adjoint", ONESHOT_ORDINARY, d_gout, n_clips, nullptr, lens, oplens, 0, nullptr, d_gin);
}

int r8bgpu_batch_oneshot_adjoint_mixed(r8bgpu_batch* b, const r8bgpu_buffer* d_gout, int n_clips, const int* plan_of_clip,
                                       const long long* lens, const long long* oplens, const r8bgpu_buffer* d_gin)
{
    return adjoint_drive(b, "batch_oneshot_adjoint_mixed", ONESHOT_MIXED, d_gout, n_clips, plan_of_clip, lens, oplens, 0, nullptr,
                         d_gin);
}

// ---- crops of long clips (include/r8bgpu.h, "crops of long clips") --------------------------------------------------

int r8bgpu_batch_oneshot_crops_adjoint(r8bgpu_batch* b, const r8bgpu_buffer* d_gout, int n_clips, const int* plan_of_clip,
                                       const long long* lens, const long long* oplens, int n_crops, const r8bgpu_crop* crops,
                                       const r8bgpu_buffer* d_gin)
{
    return adjoint_drive(b, "batch_oneshot_crops_adjoint", ONESHOT_CROPS, d_gout, n_clips, plan_of_clip, lens, oplens, n_crops, crops,
                         d_gin);
}

int r8bgpu_plan_simulate_oneshot_crops(const r8bgpu_plan* plan, int n_lanes, int n_clips, const long long* lens,
                                       const long long* oplens, int n_crops, const r8bgpu_crop* crops, int* n_calls,
                                       r8bgpu_oneshot_seg* seg, int cap)
{
    return oneshot_simulate("plan_simulate_oneshot_crops", plan, n_lanes, n_clips, lens, oplens, true, n_crops, crops, n_calls, seg,
                            cap);
}

long long r8bgpu_plan_oneshot_crop_extents(const r8bgpu_plan* plan, long long len, long long oplen, long long o0, long long o1,
                                           long long* lo, long long* hi, int cap)
{
    const char* what = "plan_oneshot_crop_extents";
    if (plan == nullptr || len < 0 || oplen < 0 || (cap > 0 && (lo == nullptr || hi == nullptr))) {
        set_err(std::string(what) + ": bad arguments");
        return -1;
    }
    if (o0 < 0 || o1 < o0 || o1 > oplen) {
        set_err(std::string(what) + ": [o0, o1) must lie within [0, oplen]");
        return -1;
    }
    const Plan& P = plan->p;
    if (const char* why = oneshot_plan_refusal(P)) {
        set_err(std::string(what) + ": " + why);
        return -1;
    }
    std::vector<std::vector<AdjPolyRec>> rec;
    AdjGeom g;
    const char* why = adjoint_records(P, len, oplen, rec);
    if (why == nullptr) why = adjoint_windows(P, std::move(rec), o0, o1, true, g);
    if (why != nullptr) {
        set_err(std::string(what) + ": " + why);
        return -1;
    }
    for (int j = 0; j < cap && j < (int) g.ext.size(); j++) {
        lo[j] = g.lo[(size_t) j];
        hi[j] = g.ext[(size_t) j];
    }
    return (long long) g.ext.size();
}

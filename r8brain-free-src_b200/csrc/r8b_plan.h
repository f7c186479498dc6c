// r8b_plan.h -- host-side resampling plan and integer "shadow scheduler".
//
// A Plan is the GPU engine's restatement of what r8b::CDSPResampler's constructor decides
// (CDSPResampler.h:117-394): which stages form the chain for (SrcSampleRate, DstSampleRate),
// their filters, and the latency bookkeeping.  Stages are expressed as operators on
// ABSOLUTELY INDEXED streams (sample n of the stage input since clear()); how many samples
// each stage has emitted after N inputs is a closed-form integer function, identical for every
// channel of a batch, so one Schedule instance drives all channels.
//
//   BlockConv (U,D)   z[q] = sum_k h[k] * xu[D*q - k],  xu[t] = x[t/U] if U|t else 0
//                     emitted(N) = max(0, ceil((U*N - Latency)/D)),  Latency = InputLen + L
//                     (CDSPBlockConvolver.h:62-185, 252-354, 512-593)
//   FracWhole         out[j] = sum_i bank[(j*InStep) % OutStep][i] * x[(j*InStep)/OutStep - fll + i]
//                     produced while  p_j + fl2 <= N-1            (CDSPFracInterpolator.h:991-1060)
//   FracPoly          order-2 interpolated bank with the resettable-counter timing
//                     (CDSPFracInterpolator.h:1069-1179, 907-919)
//   HBUp (T taps)     out[2n] = x[n]; out[2n+1] = sum_k f[k](x[n-k] + x[n+1+k]); emitted = 2*max(0,N-T)
//                     (CDSPHBUpsampler.h:674-732)
//   HBDown (T taps)   out[m] = x[2m] + sum_k f[k](x[2m+1+2k] + x[2m-1-2k]); emitted = max(0,N/2-(T-1))
//                     (CDSPHBDownsampler.h:137-239)
//
// Only the linear-phase presets are planned (fprMinPhase is out of scope, SURVEY.md section 8f).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "r8b_design.h"

namespace r8bgpu {

enum StageKind { ST_BLOCKCONV = 0, ST_FRAC_WHOLE = 1, ST_FRAC_POLY = 2, ST_HBUP = 3, ST_HBDOWN = 4 };

struct StageDesc {
    StageKind kind;
    // --- BlockConv
    int up = 1, down = 1;
    int ref_input_len = 0;   // the reference's InputLen (emission timing only)
    int latency = 0;         // the reference's Latency = InputLen + L
    int ref_prev_len = 0;    // the reference's PrevInputLen (overlap carried between its blocks)
    bool block_exact = false; // power-of-two D: the reference inverse-transforms only the lower
                             // 1/D of each block spectrum (CDSPBlockConvolver.h:329-344), which is
                             // NOT plain decimation; such stages reproduce the reference's block
                             // segmentation (FFT size 2<<BlockLenBits, blocks every InputLen).
    double norm_freq = 0, trans_band = 0, gain = 0;
    LowpassDesign lp;
    // --- Frac
    double src_rate = 0, dst_rate = 0; // as seen by this stage
    bool is_third = false;
    int in_step = 0, out_step = 0;
    bool fasttiming = false; // R8B_FASTTIMING: drifting accumulator instead of the resettable counter
    FracBank bank;
    // --- Halfband
    int hb_taps = 0;
    int steep_index = 0;
    double hb_atten = 0;
    std::vector<double> hb;
    // --- derived
    int max_out_len = 0;     // reference getMaxOutLen chain value after this stage
    int src_history = 0;     // how many source samples before "inputs so far" may be re-read
};

struct Plan {
    double src_rate = 0, dst_rate = 0;
    int max_in_len = 0;
    double trans_band = 2.0, atten = 0;
    int extfft = 0;
    int fasttiming = 0;       // R8B_FASTTIMING as given to build() (a construction parameter, whatever the chain)
    bool passthrough = false; // SrcSampleRate == DstSampleRate (CDSPResampler.h:135-138)
    std::vector<StageDesc> stages;
    int max_out_len = 0;      // CurMaxOutLen (CDSPResampler.h:502-505)
    std::string error;
    // Trim plans (build_trim): the chain's order-2 interpolator may run each channel at dst * f, |f - 1| <= max_trim.
    double max_trim = 0.0;    // 0: an ordinary plan
    int trim_stage = -1;      // index of that interpolator

    // Returns false (and sets error) for configurations this engine does not plan.  force_interp: skip the constructor's
    // shortcuts that build no interpolator (passthrough, single-step ratios, whole 2^c / 3*2^c upsampling, exact 2x / 3x
    // decimation), so that every pair gets the chain the constructor builds at a rate next to it.
    bool build(double src, double dst, int max_in_len, double tb, double atten, int phase, int extfft,
               int fasttiming, bool no_whole = false, bool force_interp = false);
    // The chain of build(src, dst, ...), except that its interpolator is always the order-2 bank (never whole
    // stepping); the buffer lengths (max_out_len per stage) are those of the largest factor 1 + max_trim.  Refuses
    // passthrough pairs and chains without an interpolator, unless any_pair forces an interpolator into every chain
    // (build(force_interp)); on the pairs it would otherwise accept, any_pair builds the same plan.
    bool build_trim(double src, double dst, int max_in_len, double tb, double atten, int extfft, double max_trim,
                    bool any_pair = false);
    // The interpolator's dsr for factor f: what build() derives at (src, fl(dst * f)) on this chain -- the product
    // rounded once, times the chain's exact power-of-two factor (1 when the interpolator ends the chain at dst).
    double trim_dsr(double f) const;
    bool trim_factor_ok(double f) const { return f >= 1.0 - max_trim && f <= 1.0 + max_trim; }

    // Test hook: a chain consisting of ONE stage, so that each kernel can be checked against the
    // corresponding reference stage class in isolation.  kind: StageKind; a[]: BLOCKCONV
    // {norm_freq, trans_band, atten, gain, up, down}; FRAC_* {src, dst, atten, is_third};
    // HBUP/HBDOWN {atten, steep_index, is_third}.
    bool build_single(int kind, const double* a, int max_in_len, int extfft);

    int in_len_before_out_pos(int req_out_pos) const; // CDSPResampler.h:406-419
    int input_required_for_output(int n) const;       // :476-484
    std::string describe() const;                      // R8BCONSOLE-style plan dump
};

// Range of absolute output indices [e0,e1) a stage emits during one process() call and the
// number of source samples [n0,n1) that became available to it.
struct StageCall {
    long long n0 = 0, n1 = 0;
    long long e0 = 0, e1 = 0;
    // FracPoly only: timing state at the first output of this call, and the rates it runs at.
    int in_counter0 = 0, in_pos_int0 = 0;
    double in_pos_shift = 0.0, fpos0 = 0.0;
    double ssr = 0.0, dsr = 0.0;
    long long p0 = 0;
    long long p_last = 0; // read position of the last output of this call (FracPoly)
    // R8B_FASTTIMING: the position sequence is inherently sequential (fpos += step with rounding), so the
    // host walks it and hands the kernel one (position - p0, fraction) pair per output of the call
    std::vector<int> ft_dp;
    std::vector<double> ft_fpos;
};

struct Schedule {
    const Plan* plan = nullptr;
    std::vector<long long> n_in, n_out; // per stage totals since clear()
    // FracPoly timing state (at most one such stage per chain, but keep per stage)
    struct PolyState {
        int in_counter = 0, in_pos_int = 0;
        double in_pos_shift = 0.0, fpos = 0.0;
        long long p = 0;
        double dsr = 0.0; // the stage's dst rate: the plan's, or the channel's trimmed one (Plan::trim_dsr)
    };
    std::vector<PolyState> poly;

    void init(const Plan* p);
    void clear(); // keeps each interpolator's dsr: a trim factor is a setting, not stream state
    // A new dsr for the trim plan's interpolator, from the next output on: the reference's own re-base
    // (CDSPFracInterpolator.h:907-919) done with the new rate, so the read position stays where it is.  Returns false
    // (and changes nothing) when dsr equals the current one bit for bit.
    bool retime(double dsr);
    // Advance by l input samples; fills one StageCall per stage; returns samples emitted by the chain.
    int advance(int l, std::vector<StageCall>& calls);
    // totals since clear(): input samples taken, output samples produced (0 for a passthrough plan, which has no stages)
    long long inputs() const { return n_in.empty() ? 0 : n_in.front(); }
    long long outputs() const { return n_out.empty() ? 0 : n_out.back(); }
};

// End of a stream: what CDSPResampler::oneshot() does after the last real input sample (CDSPResampler.h:592-651) --
// silence is fed until the stream's output reaches `target` (absolute output index since clear()), the samples from
// the current output position up to `target` are returned, and the stream is then cleared.  The silence goes in as
// the smallest length that reaches the target, cut into sub-steps of at most MaxInLen; the last stage of the last
// sub-step stops at `target` (see plan_flush for the half-band upsampler).  Chunking changes only the rounding of the values (DESIGN.md section 7), never the
// counts: count = max(0, target - outputs produced so far).
struct FlushPlan {
    long long target = 0;
    long long zeros = 0;                         // silence fed (0 when the target is already reached)
    int count = 0;                               // samples returned
    std::vector<int> lens;                       // sub-step lengths
    std::vector<std::vector<StageCall>> calls;   // per sub-step: one StageCall per stage
};
// Plans the flush of a stream in state s (not a passthrough plan); count must fit an int (the caller checks it first).
// keep_calls = false: counts and lengths only (a dry run), no StageCalls are kept.  A half-band upsampler as the last
// stage writes outputs in pairs: its last range then ends at the target rounded up to even, one sample past `count`.
void plan_flush(const Schedule& s, long long target, FlushPlan& f, bool keep_calls = true);
// ceil(n_in * dst / src), computed exactly on the binary values of the two rates; -1 when it exceeds LLONG_MAX.
long long flush_default_target(const Plan& p, long long n_in);
// Upper bound of max(0, flush_default_target(N) - outputs(N)) over every N and every chunking (r8b_plan.cpp).
int flush_max_out_len(const Plan& p);

// Two schedules are equal when every later call advances them alike (same totals and order-2 timing state).
bool same_state(const Schedule& a, const Schedule& b);

// The schedules of a batch whose channels have diverged: ragged calls gave them different block lengths, or some of them
// were cleared on their own.  Channels whose schedules are equal share one group, so a batch whose channels all received
// the same lengths since their last clear has one group (and runs in lock-step again).
struct RaggedSchedule {
    std::vector<Schedule> groups;
    std::vector<int> group_of; // per channel

    // One call, planned without changing the state: every distinct (group, block length) pair is a key with its own
    // StageCalls; a run is a range of consecutive channels with the same key.
    struct Run {
        int c0, n, key;
    };
    struct Step {
        std::vector<Schedule> next;                  // per key: the schedule after the call
        std::vector<int> len, count;                 // per key: block length, samples produced
        std::vector<std::vector<StageCall>> calls;   // per key
        std::vector<int> key_of;                     // per channel
        std::vector<Run> runs;
    };

    void init(const Schedule& lockstep, int n_ch); // every channel in the state `lockstep`
    void plan_call(const int* lens, Step& step) const;
    void commit(const Step& step);
    void clear_channels(const int* ch, int n);       // the named channels return to the state after clear()
    void retime_channels(const int* ch, int n, const double* dsr); // Schedule::retime on the named channels
    void install(const int* ch, int n, const Schedule* s); // channel ch[i] takes the state s[i] (an imported stream)
    bool converged() const { return groups.size() == 1; }
    const Schedule& of(int c) const { return groups[(size_t) group_of[(size_t) c]]; }

private:
    void merge(std::vector<Schedule>& g, std::vector<int>& of); // fold equal schedules into one group
};

// emitted-sample count helpers (exposed for tests)
long long blockconv_emitted(const StageDesc& s, long long n_in);
long long frac_whole_emitted(const StageDesc& s, long long n_in);
long long hbup_emitted(const StageDesc& s, long long n_in);
long long hbdown_emitted(const StageDesc& s, long long n_in);

} // namespace r8bgpu

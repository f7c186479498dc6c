// include/r8b/CDSPResampler.h -- header-style C++ front-end in namespace r8b over the r8bgpu C-ABI.
//
// Drop-in for the reference's CDSPResampler.h on the process() path: same class names,
// constructor arguments, method names and ownership rules (CDSPResampler.h:117-651,729-810 of
// avaneev/r8brain-free-src); the per-channel CPU pipeline behind them is replaced by sm_90a
// kernels reached through include/r8bgpu.h.  Link with -lr8bgpu.
//
//   r8b::CDSPResampler / CDSPResampler16 / CDSPResampler16IR / CDSPResampler24
//        one stream per object, HOST buffers; process() = H2D + kernels + D2H per call.
//        Meant for drop-in correctness; it cannot be fast (one PCIe round trip per call).
//   r8b::CDSPResamplerBatch (new)
//        N independent channels processed in lock-step -- the shape of example.cpp:30-67 --
//        with host OR device planar buffers.  This is the intended production entry.
//
// Configuration macros (r8bconf.h surface).  The FFT back-end selectors R8B_IPP, R8B_PFFFT,
// R8B_PFFFT_DOUBLE, R8B_FLOATFFT are accepted and ignored (there is no CPU FFT and no CPU
// fallback).  R8B_EXTFFT and R8B_FASTTIMING change the plan exactly as they change the reference
// (block length -> emission latency; interpolator timing) and are forwarded to the planner.
// R8BASSERT / R8BCONSOLE keep their meaning (no-ops unless defined by the user).
#ifndef R8B_CDSPRESAMPLER_B200_INCLUDED
#define R8B_CDSPRESAMPLER_B200_INCLUDED

#include <cstddef>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <vector>

#include "../r8bgpu.h"

#ifndef R8B_EXTFFT
#define R8B_EXTFFT 0
#endif
#ifndef R8B_FASTTIMING
#define R8B_FASTTIMING 0
#endif
#ifndef R8BASSERT
#define R8BASSERT(e)
#endif
#ifndef R8BCONSOLE
#define R8BCONSOLE(...)
#endif

namespace r8b {

/// Filter phase response (CDSPFIRFilter.h:34-46).  Only fprLinearPhase is implemented.
enum EDSPFilterPhaseResponse { fprLinearPhase = 0, fprMinPhase = 1 };

/// N channels resampled in lock-step on one GPU.
class CDSPResamplerBatch {
public:
    CDSPResamplerBatch(const int NumChannels, const double SrcSampleRate, const double DstSampleRate,
                       const int aMaxInLen, const double ReqTransBand = 2.0, const double ReqAtten = 206.91,
                       const EDSPFilterPhaseResponse ReqPhase = fprLinearPhase, const int Device = -1)
        : Plan(r8bgpu_plan_create(SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, ReqAtten,
                                  (int) ReqPhase, R8B_EXTFFT, R8B_FASTTIMING))
        , Batch(NULL)
        , Channels(NumChannels)
        , Dev(Device)
        , MaxInLen(aMaxInLen)
        , PlanSrc(1, SrcSampleRate)
        , PlanDst(1, DstSampleRate)
    {
        R8BASSERT(Plan != NULL);
        if (Plan != NULL) {
            char buf[1024];
            r8bgpu_plan_describe(Plan, buf, (int) sizeof(buf));
            R8BCONSOLE("%s", buf);
            (void) buf;
        }
    }

    /// Independent streams at different rates in one batch (r8bgpu_batch_create_mixed): channel c is resampled from
    /// SrcRates[c] to DstRates[c], as its own CDSPResampler would be.  One plan is made per distinct (src, dst) pair.
    /// processRagged / processRaggedDevice, clearChannels, flushChannels / flushChannelsDevice and the batched oneshot()
    /// work per channel; the lock-step process() calls are refused.  getMaxOutLen() / getFlushMaxOutLen() are the
    /// largest values of the plans.
    CDSPResamplerBatch(const int NumChannels, const double* SrcRates, const double* DstRates, const int aMaxInLen,
                       const double ReqTransBand, const double ReqAtten, const int Device = R8BGPU_DEVICE_CURRENT)
        : Plan(NULL)
        , Batch(NULL)
        , Channels(NumChannels)
        , Dev(Device)
        , MaxInLen(aMaxInLen)
    {
        std::vector<double> Src, Dst;
        for (int c = 0; c < NumChannels; c++) {
            size_t p = 0;
            while (p < Src.size() && !(Src[p] == SrcRates[c] && Dst[p] == DstRates[c])) p++;
            if (p == Src.size()) {
                Src.push_back(SrcRates[c]);
                Dst.push_back(DstRates[c]);
                r8bgpu_plan* h = r8bgpu_plan_create(SrcRates[c], DstRates[c], aMaxInLen, ReqTransBand, ReqAtten,
                                                    (int) fprLinearPhase, R8B_EXTFFT, R8B_FASTTIMING);
                if (h == NULL) Failed = true;
                Plans.push_back(h);
            }
            PlanOf.push_back((int) p);
        }
        PlanSrc = Src;
        PlanDst = Dst;
        R8BASSERT(!Failed);
    }

    /// Drift compensation (r8bgpu_plan_create_trim): every channel's ratio may be trimmed by its own factor f in
    /// [1 - MaxTrim, 1 + MaxTrim] (0 < MaxTrim <= 0.01) with setRateTrim(); channel c then produces about
    /// DstSampleRate * f samples per SrcSampleRate inputs.  The chain's interpolator is always the order-2 bank.
    /// Flushes take explicit targets only.  AnyPair (r8bgpu_plan_create_asrc) accepts every rate pair, SrcSampleRate ==
    /// DstSampleRate and integer ratios included, which the reference otherwise plans without an interpolator.
    CDSPResamplerBatch(const int NumChannels, const double SrcSampleRate, const double DstSampleRate,
                       const int aMaxInLen, const double ReqTransBand, const double ReqAtten, const double MaxTrim,
                       const int Device = -1, const bool AnyPair = false)
        : Plan((AnyPair ? r8bgpu_plan_create_asrc : r8bgpu_plan_create_trim)(SrcSampleRate, DstSampleRate, aMaxInLen,
                                                                            ReqTransBand, ReqAtten, R8B_EXTFFT, MaxTrim))
        , Batch(NULL)
        , Channels(NumChannels)
        , Dev(Device)
        , MaxInLen(aMaxInLen)
        , PlanSrc(1, SrcSampleRate)
        , PlanDst(1, DstSampleRate)
    {
        R8BASSERT(Plan != NULL);
    }

    /// Trim factors of the named channels, from each one's next call on (r8bgpu_batch_set_trim); returns 0 or -1.
    int setRateTrim(const int* Chans, const int n, const double* Factors)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_set_trim(Batch, Chans, n, Factors);
    }

    /// Dithered integer output for the named channels (r8bgpu_batch_set_dither): Cfg[i] for channel Chans[i], OFF (the
    /// plain cast) or TPDF with optional error-feedback taps.  Settings survive clear(); returns 0 or -1.
    int setDither(const int* Chans, const int n, const r8bgpu_dither* Cfg)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_set_dither(Batch, Chans, n, Cfg);
    }

    /// Every channel's trim factor (getNumChannels() entries; 1 for channels of an ordinary plan); returns 0 or -1.
    int getRateTrim(double* Factors)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_trim(Batch, Factors);
    }

    ~CDSPResamplerBatch()
    {
        if (Batch != NULL) r8bgpu_batch_destroy(Batch);
        if (Plan != NULL) r8bgpu_plan_destroy(Plan);
        for (size_t p = 0; p < Plans.size(); p++)
            if (Plans[p] != NULL) r8bgpu_plan_destroy(Plans[p]);
    }

    /// false: the constructor arguments were refused (out-of-range parameters, fprMinPhase ...) or, after the first
    /// call, no CUDA device / no memory for the batch.  The reference has no such state (R8BASSERT compiles out and
    /// bad parameters are undefined behaviour); here every accessor of an invalid object returns 0 and every
    /// process() returns -1, and getLastError() says why.
    bool isValid() const { return (Plan != NULL || !Plans.empty()) && !Failed; }
    const char* getLastError() const { return r8bgpu_last_error(); }
    int getNumChannels() const { return Channels; }
    int getMaxOutLen(const int /* MaxInLen */ = 0) const
    {
        if (Plan != NULL) return r8bgpu_plan_max_out_len(Plan);
        int m = 0; // a mixed batch: the largest of its plans' (r8bgpu_batch_max_out_len)
        for (size_t p = 0; p < Plans.size(); p++)
            if (Plans[p] != NULL) m = std::max(m, r8bgpu_plan_max_out_len(Plans[p]));
        return m;
    }
    int getInLenBeforeOutPos(const int ReqOutPos) const { return Plan ? r8bgpu_plan_in_len_before_out_pos(Plan, ReqOutPos) : 0; }
    int getInputRequiredForOutput(const int ReqOutSamples) const { return Plan ? r8bgpu_plan_input_required_for_output(Plan, ReqOutSamples) : 0; }
    int getLatency() const { return 0; }
    double getLatencyFrac() const { return Plan ? r8bgpu_plan_latency_frac(Plan) : 0.0; }

    void clear()
    {
        if (Batch != NULL) r8bgpu_batch_clear(Batch);
    }

    /// Host planar buffers: channel c at ip + c*InStride / op + c*OutStride (strides in doubles).
    /// Returns samples written per channel (same for all channels), or -1.
    int process(const double* ip, const size_t InStride, const int l, double* op, const size_t OutStride,
                const int OutCap)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_process_host(Batch, ip, InStride, l, op, OutStride, OutCap);
    }

    /// Device planar buffers; asynchronous on the batch stream (see r8bgpu_batch_set_stream()).
    int processDevice(const double* d_ip, const size_t InStride, const int l, double* d_op, const size_t OutStride,
                      const int OutCap)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_process(Batch, d_ip, InStride, l, d_op, OutStride, OutCap);
    }

    /// Typed buffers (int16 / packed int24 / int32 / float32 / float64, planar or interleaved): the
    /// sample conversions of oneshot<Tin,Tout>() (CDSPResampler.h:592-651) run on the device.
    int process(const r8bgpu_buffer& ip, const int l, const r8bgpu_buffer& op, const int OutCap)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_process_host_fmt(Batch, &ip, l, &op, OutCap);
    }

    int processDevice(const r8bgpu_buffer& d_ip, const int l, const r8bgpu_buffer& d_op, const int OutCap)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_process_fmt(Batch, &d_ip, l, &d_op, OutCap);
    }

    /// Independent streams: channel c takes lens[c] samples (0..MaxInLen) this call and writes counts[c] samples, as
    /// if each channel were its own CDSPResampler.  Host planar buffers; returns 0 or -1.
    int processRagged(const double* ip, const size_t InStride, const int* lens, double* op, const size_t OutStride,
                      const int OutCap, int* counts)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_process_host_ragged(Batch, ip, InStride, lens, op, OutStride, OutCap, counts);
    }

    /// Device planar buffers; asynchronous on the batch stream, counts[] is filled when the call returns.
    int processRaggedDevice(const double* d_ip, const size_t InStride, const int* lens, double* d_op,
                            const size_t OutStride, const int OutCap, int* counts)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_process_ragged(Batch, d_ip, InStride, lens, d_op, OutStride, OutCap, counts);
    }

    /// Independent streams with typed host buffers (planar or interleaved; the conversions of oneshot<Tin,Tout>()
    /// run on the device).  Returns 0 or -1.
    int processRagged(const r8bgpu_buffer& ip, const int* lens, const r8bgpu_buffer& op, const int OutCap, int* counts)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_process_host_ragged_fmt(Batch, &ip, lens, &op, OutCap, counts);
    }

    /// Typed device buffers; asynchronous on the batch stream, counts[] is filled when the call returns.
    int processRaggedDevice(const r8bgpu_buffer& d_ip, const int* lens, const r8bgpu_buffer& d_op, const int OutCap,
                            int* counts)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_process_ragged_fmt(Batch, &d_ip, lens, &d_op, OutCap, counts);
    }

    /// clear() of the named channels only (CDSPResampler.h:521-529 per channel object); returns 0 or -1.
    int clearChannels(const int* Channels, const int n)
    {
        return Batch != NULL ? r8bgpu_batch_clear_channels(Batch, Channels, n) : 0;
    }

    /// Moving streams (r8bgpu_batch_export / _import): the complete state of channel Chans[i] as a blob at
    /// Buf + i * Stride (host memory; Device = true: device memory on the batch's GPU).  Importing a blob into any slot of
    /// a batch of the same plan continues the stream there bit for bit.  getStateBytes(c): the blob size of channel c's
    /// plan.  Return 0 or -1.
    int exportChannels(const int* Chans, const int n, void* Buf, const size_t Stride, const bool Device = false)
    {
        if (!ensure()) return -1;
        return Device ? r8bgpu_batch_export_device(Batch, Chans, n, Buf, Stride) : r8bgpu_batch_export(Batch, Chans, n, Buf, Stride);
    }
    int importChannels(const int* Chans, const int n, const void* Buf, const size_t Stride, const bool Device = false)
    {
        if (!ensure()) return -1;
        return Device ? r8bgpu_batch_import_device(Batch, Chans, n, Buf, Stride) : r8bgpu_batch_import(Batch, Chans, n, Buf, Stride);
    }
    size_t getStateBytes(const int Chan = 0) const
    {
        if (Plan != NULL) return r8bgpu_plan_state_bytes(Plan);
        return Chan >= 0 && (size_t) Chan < PlanOf.size() ? r8bgpu_plan_state_bytes(Plans[(size_t) PlanOf[(size_t) Chan]]) : 0;
    }

    /// End of stream for the named channels: the silence-feeding tail of oneshot() (CDSPResampler.h:592-651), then
    /// clear().  Targets (NULL: ceil(inputs * Dst / Src)) are output counts since each channel's last clear; counts[c]
    /// receives the samples written for every channel (0 for those not named).  Size OutCap with getFlushMaxOutLen().
    /// Host planar buffers; returns 0 or -1.  See r8bgpu_batch_flush_host().
    int flushChannels(const int* Chans, const int n, const long long* Targets, double* op, const size_t OutStride,
                      const int OutCap, int* counts)
    {
        const r8bgpu_buffer o = {op, R8BGPU_F64, 0, OutStride, 1.0};
        return flushChannels(Chans, n, Targets, o, OutCap, counts);
    }

    /// Typed host buffers (any format, planar or interleaved).
    int flushChannels(const int* Chans, const int n, const long long* Targets, const r8bgpu_buffer& op, const int OutCap,
                      int* counts)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_flush_host(Batch, Chans, n, Targets, &op, OutCap, counts);
    }

    /// Device buffers; asynchronous on the batch stream, counts[] is filled when the call returns.
    int flushChannelsDevice(const int* Chans, const int n, const long long* Targets, double* d_op, const size_t OutStride,
                            const int OutCap, int* counts)
    {
        const r8bgpu_buffer o = {d_op, R8BGPU_F64, 0, OutStride, 1.0};
        return flushChannelsDevice(Chans, n, Targets, o, OutCap, counts);
    }

    int flushChannelsDevice(const int* Chans, const int n, const long long* Targets, const r8bgpu_buffer& d_op,
                            const int OutCap, int* counts)
    {
        if (!ensure()) return -1;
        return r8bgpu_batch_flush(Batch, Chans, n, Targets, &d_op, OutCap, counts);
    }

    /// Upper bound of what a default-target flush returns per channel.
    int getFlushMaxOutLen() const
    {
        if (Plan != NULL) return r8bgpu_plan_flush_max_out_len(Plan);
        int m = 0; // a mixed batch: the largest of its plans' (r8bgpu_batch_flush_max_out_len)
        for (size_t p = 0; p < Plans.size(); p++)
            if (Plans[p] != NULL) m = std::max(m, r8bgpu_plan_flush_max_out_len(Plans[p]));
        return m;
    }

    /// Batched oneshot() over a padded host batch: per channel exactly the reference's
    /// oneshot(ip + c*InStride, lens[c], op + c*OutStride, oplens[c]) (CDSPResampler.h:592-651) on a fresh object.
    /// Every channel is cleared first; the clips go in as ragged calls of at most MaxInLen samples, then one flush
    /// completes every clip at oplens[c].  The batch is left cleared.  Returns 0 or -1.
    int oneshot(const double* ip, const size_t InStride, const int* lens, double* op, const size_t OutStride,
                const int* oplens)
    {
        if (!ensure() || r8bgpu_batch_clear(Batch) != 0) return -1;
        const int Cap = getMaxOutLen() > 0 ? getMaxOutLen() : 1;
        std::vector<double> Blk((size_t) Channels * (size_t) Cap);
        std::vector<int> Lens((size_t) Channels), Counts((size_t) Channels), Pos((size_t) Channels, 0);
        int MaxLen = 0;
        for (int c = 0; c < Channels; c++) MaxLen = std::max(MaxLen, lens[c]);
        for (int Off = 0; Off < MaxLen; Off += MaxInLen) {
            for (int c = 0; c < Channels; c++) Lens[(size_t) c] = std::max(0, std::min(MaxInLen, lens[c] - Off));
            if (r8bgpu_batch_process_host_ragged(Batch, ip + Off, InStride, &Lens[0], &Blk[0], (size_t) Cap, Cap, &Counts[0]) != 0)
                return -1;
            for (int c = 0; c < Channels; c++) { // as oneshot(): nothing past oplen is kept
                const int Take = std::min(Counts[(size_t) c], oplens[c] - Pos[(size_t) c]);
                if (Take > 0) std::copy(Blk.begin() + (size_t) c * Cap, Blk.begin() + (size_t) c * Cap + Take, op + c * OutStride + Pos[(size_t) c]);
                Pos[(size_t) c] += std::max(0, Take);
            }
        }
        std::vector<int> All((size_t) Channels);
        std::vector<long long> Targets((size_t) Channels);
        int Tail = 1;
        for (int c = 0; c < Channels; c++) {
            All[(size_t) c] = c;
            Targets[(size_t) c] = oplens[c];
            Tail = std::max(Tail, oplens[c] - Pos[(size_t) c]);
        }
        std::vector<double> TailBuf((size_t) Channels * (size_t) Tail);
        if (flushChannels(&All[0], Channels, &Targets[0], &TailBuf[0], (size_t) Tail, Tail, &Counts[0]) != 0) return -1;
        for (int c = 0; c < Channels; c++)
            std::copy(TailBuf.begin() + (size_t) c * Tail, TailBuf.begin() + (size_t) c * Tail + Counts[(size_t) c],
                      op + c * OutStride + Pos[(size_t) c]);
        return 0;
    }

    /// Whole clips on every channel of the batch used as a lane (r8bgpu_batch_oneshot_host, include/r8bgpu.h "long
    /// clips"): clip r is ip + r*InStride (lens[r] samples, 64-bit) and its output op + r*OutStride (oplens[r]
    /// samples; oplens NULL: ceil(lens[r] * dst / src)), bit for bit what oneshot() above returns for that clip on a
    /// one-channel batch, for any number of clips.  The batch is cleared before and after.  Returns 0 or -1.
    int oneshotLong(const double* ip, const size_t InStride, int NumClips, const long long* lens, double* op,
                    const size_t OutStride, const long long* oplens)
    {
        if (!ensure()) return -1;
        r8bgpu_buffer In = {const_cast<double*>(ip), R8BGPU_F64, 0, InStride, 1.0};
        r8bgpu_buffer Out = {op, R8BGPU_F64, 0, OutStride, 1.0};
        return r8bgpu_batch_oneshot_host(Batch, &In, NumClips, lens, &Out, oplens, NULL) == 0 ? 0 : -1;
    }

    /// The transpose of oneshotLong for gradients (r8bgpu_batch_oneshot_adjoint, include/r8bgpu.h "gradients through
    /// long clips"), on DEVICE buffers: clip r's output gradient is d_gout + r*GoutStride (oplens[r] samples; NULL:
    /// ceil(lens[r] * dst / src)) and its input gradient d_gin + r*GinStride (lens[r] samples).  Returns 0 or -1.
    int oneshotLongAdjoint(const double* d_gout, const size_t GoutStride, int NumClips, const long long* lens,
                           const long long* oplens, double* d_gin, const size_t GinStride)
    {
        if (!ensure()) return -1;
        r8bgpu_buffer G = {const_cast<double*>(d_gout), R8BGPU_F64, 0, GoutStride, 1.0};
        r8bgpu_buffer X = {d_gin, R8BGPU_F64, 0, GinStride, 1.0};
        return r8bgpu_batch_oneshot_adjoint(Batch, &G, NumClips, lens, oplens, &X) == 0 ? 0 : -1;
    }

    /// oneshotLong for clips at mixed rates (r8bgpu_batch_oneshot_mixed_host, include/r8bgpu.h "long clips at mixed
    /// rates"): clip r is resampled from ClipSrcRates[r] to ClipDstRates[r] on the lanes of the channels made for that
    /// pair by the rates constructor, bit for bit as oneshotLong on a batch of that pair alone (oplens NULL: each clip's
    /// ceil(lens[r] * dst / src)).  A pair the batch has no channel for is refused.  Returns 0 or -1.
    int oneshotLong(const double* ip, const size_t InStride, int NumClips, const double* ClipSrcRates,
                    const double* ClipDstRates, const long long* lens, double* op, const size_t OutStride,
                    const long long* oplens)
    {
        std::vector<int> PlanOfClip;
        if (!ensure()) return -1;
        clipPlans(NumClips, ClipSrcRates, ClipDstRates, PlanOfClip);
        r8bgpu_buffer In = {const_cast<double*>(ip), R8BGPU_F64, 0, InStride, 1.0};
        r8bgpu_buffer Out = {op, R8BGPU_F64, 0, OutStride, 1.0};
        return r8bgpu_batch_oneshot_mixed_host(Batch, &In, NumClips, PlanOfClip.empty() ? NULL : &PlanOfClip[0], lens, &Out,
                                               oplens, NULL) == 0 ? 0 : -1;
    }

    /// oneshotLongAdjoint for clips at mixed rates (r8bgpu_batch_oneshot_adjoint_mixed), on DEVICE buffers, with the
    /// per-clip rate pairs of the oneshotLong overload above.  Returns 0 or -1.
    int oneshotLongAdjoint(const double* d_gout, const size_t GoutStride, int NumClips, const double* ClipSrcRates,
                           const double* ClipDstRates, const long long* lens, const long long* oplens, double* d_gin,
                           const size_t GinStride)
    {
        std::vector<int> PlanOfClip;
        if (!ensure()) return -1;
        clipPlans(NumClips, ClipSrcRates, ClipDstRates, PlanOfClip);
        r8bgpu_buffer G = {const_cast<double*>(d_gout), R8BGPU_F64, 0, GoutStride, 1.0};
        r8bgpu_buffer X = {d_gin, R8BGPU_F64, 0, GinStride, 1.0};
        return r8bgpu_batch_oneshot_adjoint_mixed(Batch, &G, NumClips, PlanOfClip.empty() ? NULL : &PlanOfClip[0], lens,
                                                  oplens, &X) == 0 ? 0 : -1;
    }

    /// Crops of long clips (r8bgpu_batch_oneshot_crops_host, include/r8bgpu.h "crops of long clips"), host buffers:
    /// crop k (clip, outputs [o0, o1)) goes to op + k*OutStride, bit for bit outputs [o0, o1) of oneshotLong's output
    /// for that clip; only the crops' spans run.  oplens NULL: each clip's ceil(lens[r] * dst / src).  Returns 0 or -1.
    int oneshotCrops(const double* ip, const size_t InStride, int NumClips, const long long* lens, const long long* oplens,
                     int NumCrops, const r8bgpu_crop* crops, double* op, const size_t OutStride)
    {
        if (!ensure()) return -1;
        r8bgpu_buffer In = {const_cast<double*>(ip), R8BGPU_F64, 0, InStride, 1.0};
        r8bgpu_buffer Out = {op, R8BGPU_F64, 0, OutStride, 1.0};
        return r8bgpu_batch_oneshot_crops_host(Batch, &In, NumClips, NULL, lens, oplens, NumCrops, crops, &Out, NULL) == 0 ? 0
                                                                                                                           : -1;
    }

    /// oneshotCrops for clips at mixed rates: clip r from ClipSrcRates[r] to ClipDstRates[r], as the per-clip-rate
    /// oneshotLong overload.  Returns 0 or -1.
    int oneshotCrops(const double* ip, const size_t InStride, int NumClips, const double* ClipSrcRates,
                     const double* ClipDstRates, const long long* lens, const long long* oplens, int NumCrops,
                     const r8bgpu_crop* crops, double* op, const size_t OutStride)
    {
        std::vector<int> PlanOfClip;
        if (!ensure()) return -1;
        clipPlans(NumClips, ClipSrcRates, ClipDstRates, PlanOfClip);
        r8bgpu_buffer In = {const_cast<double*>(ip), R8BGPU_F64, 0, InStride, 1.0};
        r8bgpu_buffer Out = {op, R8BGPU_F64, 0, OutStride, 1.0};
        return r8bgpu_batch_oneshot_crops_host(Batch, &In, NumClips, PlanOfClip.empty() ? NULL : &PlanOfClip[0], lens, oplens,
                                               NumCrops, crops, &Out, NULL) == 0 ? 0 : -1;
    }

    void setStream(void* CudaStream)
    {
        if (ensure()) r8bgpu_batch_set_stream(Batch, CudaStream);
    }

    void sync()
    {
        if (Batch != NULL) r8bgpu_batch_sync(Batch);
    }

    r8bgpu_batch* handle()
    {
        ensure();
        return Batch;
    }

private:
    r8bgpu_plan* Plan;
    r8bgpu_batch* Batch;
    int Channels;
    int Dev;
    int MaxInLen;
    bool Failed = false; // batch creation was tried and refused: do not retry on every call
    std::vector<r8bgpu_plan*> Plans; // a mixed batch: one plan per distinct rate pair, PlanOf[c] = channel c's
    std::vector<int> PlanOf;
    std::vector<double> PlanSrc, PlanDst; // the rate pair of each plan (an ordinary batch: its one plan, index 0)

    // Each clip's plan index from its rate pair: -1 for a pair without a plan and a null PlanOfClip for null rates,
    // which the C-ABI refuses with its message.
    void clipPlans(int NumClips, const double* Src, const double* Dst, std::vector<int>& PlanOfClip) const
    {
        if (Src == NULL || Dst == NULL) return;
        for (int r = 0; r < NumClips; r++) {
            size_t p = 0;
            while (p < PlanSrc.size() && !(PlanSrc[p] == Src[r] && PlanDst[p] == Dst[r])) p++;
            PlanOfClip.push_back(p < PlanSrc.size() ? (int) p : -1);
        }
    }

    bool ensure()
    {
        if (Batch == NULL && Plan != NULL && !Failed) {
            Batch = r8bgpu_batch_create(Plan, Channels, Dev);
            Failed = (Batch == NULL);
        } else if (Batch == NULL && !Plans.empty() && !Failed) {
            Batch = r8bgpu_batch_create_mixed(&Plans[0], (int) Plans.size(), &PlanOf[0], Channels, Dev);
            Failed = (Batch == NULL);
        }
        R8BASSERT(Batch != NULL);
        return Batch != NULL;
    }

    CDSPResamplerBatch(const CDSPResamplerBatch&);
    CDSPResamplerBatch& operator=(const CDSPResamplerBatch&);
};

/// "Pull" use of a batch for real-time callers (README.md:132-146 of the reference: "a pull method ... calls the
/// resampling process until the output buffer is filled", keeping the excess output for the next request).  The
/// reference leaves that loop to the caller; this helper is the same loop around CDSPResamplerBatch with host buffers:
/// pull() asks `fill` for input blocks of at most MaxInLen frames per channel until `n` output frames per channel are
/// available, hands them out, and keeps what is left over.  Output is exactly the push-mode stream, in the same order.
class CDSPResamplerPull {
public:
    CDSPResamplerPull(const int NumChannels, const double SrcSampleRate, const double DstSampleRate, const int aMaxInLen,
                      const double ReqTransBand = 2.0, const double ReqAtten = 206.91, const int Device = -1)
        : Rs(NumChannels, SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, ReqAtten, fprLinearPhase, Device)
        , Channels(NumChannels)
        , MaxInLen(aMaxInLen)
        , Cap(Rs.getMaxOutLen() > 0 ? Rs.getMaxOutLen() : 1)
        , Have(0)
        , In((size_t) NumChannels * (size_t) aMaxInLen)
        , Out((size_t) NumChannels * (size_t) Cap)
        , Fifo((size_t) NumChannels)
    {
    }

    bool isValid() const { return Rs.isValid(); }
    CDSPResamplerBatch& batch() { return Rs; }

    /// fill(double* ip, size_t stride, int maxFrames) -> frames written per channel (planar, channel c at ip + c*stride);
    /// returning 0 ends the stream (pull() then returns fewer than n frames).  op: planar, channel c at op + c*OutStride.
    template <typename Fill>
    int pull(Fill fill, double* op, const size_t OutStride, const int n)
    {
        while (Have < n) {
            const int l = fill(&In[0], (size_t) MaxInLen, MaxInLen);
            if (l <= 0) break;
            const int got = Rs.process(&In[0], (size_t) MaxInLen, l, &Out[0], (size_t) Cap, Cap);
            if (got < 0) return -1;
            for (int c = 0; c < Channels; c++)
                Fifo[(size_t) c].insert(Fifo[(size_t) c].end(), Out.begin() + (size_t) c * Cap, Out.begin() + (size_t) c * Cap + got);
            Have += got;
        }
        const int give = Have < n ? Have : n;
        for (int c = 0; c < Channels; c++) {
            std::vector<double>& f = Fifo[(size_t) c];
            std::copy(f.begin(), f.begin() + give, op + (size_t) c * OutStride);
            f.erase(f.begin(), f.begin() + give);
        }
        Have -= give;
        return give;
    }

    void clear()
    {
        Rs.clear();
        for (size_t c = 0; c < Fifo.size(); c++) Fifo[c].clear();
        Have = 0;
    }

private:
    CDSPResamplerBatch Rs;
    int Channels, MaxInLen, Cap, Have;
    std::vector<double> In, Out;
    std::vector<std::vector<double> > Fifo;
};

/// Single-stream object with the reference's exact call shape.
class CDSPResampler {
public:
    CDSPResampler(const double SrcSampleRate, const double DstSampleRate, const int aMaxInLen,
                  const double ReqTransBand = 2.0, const double ReqAtten = 206.91,
                  const EDSPFilterPhaseResponse ReqPhase = fprLinearPhase)
        : Impl(1, SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, ReqAtten, ReqPhase)
        , MaxInLen(aMaxInLen)
        , IsSame(SrcSampleRate == DstSampleRate)
    {
        R8BASSERT(SrcSampleRate > 0.0);
        R8BASSERT(DstSampleRate > 0.0);
        R8BASSERT(aMaxInLen > 0);
        OutBuf.resize((size_t) (Impl.getMaxOutLen() > 0 ? Impl.getMaxOutLen() : 1));
    }

    virtual ~CDSPResampler() {}

    /// Not in the reference: see CDSPResamplerBatch::isValid().  An invalid object produces no output: process()
    /// returns 0 samples, oneshot() zero-fills, getInLenBeforeOutStart() returns 0 -- none of them loops.
    bool isValid() const { return IsSame || (Impl.isValid() && !Broken); }
    const char* getLastError() const { return Impl.getLastError(); }

    virtual int getInLenBeforeOutPos(const int ReqOutPos) const { return Impl.getInLenBeforeOutPos(ReqOutPos); }
    int getInputRequiredForOutput(const int ReqOutSamples) const { return Impl.getInputRequiredForOutput(ReqOutSamples); }
    virtual int getLatency() const { return 0; }
    virtual double getLatencyFrac() const { return Impl.getLatencyFrac(); }
    virtual int getMaxOutLen(const int /* MaxInLen */) const { return Impl.getMaxOutLen(); }
    virtual void clear() { Impl.clear(); }

    /// As CDSPResampler.h:443-464: feeds single samples until the output passes ReqOutPos.
    int getInLenBeforeOutStart(const int ReqOutPos = 0)
    {
        int inc = 0, outc = 0;
        while (true) {
            double ins = 0.0;
            double* op;
            outc += process(&ins, 1, op);
            if (!isValid()) return 0; // a failed object never produces output: do not spin
            if (outc > ReqOutPos) {
                clear();
                return inc;
            }
            inc++;
        }
    }

    /// As CDSPResampler.h:559-575: `op0` receives a pointer to an internal buffer that stays valid
    /// until the next call; the input is never written; equal rates hand the input back.
    virtual int process(double* ip0, int l, double*& op0)
    {
        R8BASSERT(l >= 0);
        if (IsSame) {
            op0 = ip0;
            return l;
        }
        op0 = &OutBuf[0];
        const int n = Impl.process(ip0, (size_t) l, l, op0, OutBuf.size(), (int) OutBuf.size());
        R8BASSERT(n >= 0);
        if (n < 0) Broken = true; // sticky: isValid() turns false, the loops below stop
        return n < 0 ? 0 : n;
    }

    /// One-shot conversion of a whole signal (semantics of CDSPResampler.h:592-651): the input is fed in
    /// MaxInLen-sized pieces, followed by silence, until `oplen` output samples have been collected; the
    /// stream state is cleared afterwards.  Tin/Tout may be any arithmetic sample type.
    template <typename Tin, typename Tout>
    void oneshot(const Tin* ip, int iplen, Tout* op, int oplen)
    {
        std::vector<double> chunk((size_t) MaxInLen, 0.0);
        int fed = 0, got = 0;
        while (got < oplen) {
            const int n = (fed < iplen) ? ((iplen - fed < MaxInLen) ? iplen - fed : MaxInLen) : MaxInLen;
            if (fed < iplen) {
                for (int i = 0; i < n; i++) chunk[(size_t) i] = (double) ip[fed + i];
                fed += n;
                if (fed >= iplen && n < MaxInLen) std::fill(chunk.begin() + n, chunk.end(), 0.0);
            } else if (fed == iplen) {
                std::fill(chunk.begin(), chunk.end(), 0.0); // from here on: silence
                fed++;
            }
            double* res = NULL;
            int produced = process(&chunk[0], n, res);
            if (!isValid()) { // no device, refused parameters, launch failure: silence instead of an endless loop
                for (int i = got; i < oplen; i++) op[i] = (Tout) 0;
                return;
            }
            if (produced > oplen - got) produced = oplen - got;
            for (int i = 0; i < produced; i++) op[got + i] = (Tout) res[i];
            got += produced;
        }
        clear();
    }

private:
    CDSPResamplerBatch Impl;
    std::vector<double> OutBuf;
    int MaxInLen;
    bool IsSame;
    bool Broken = false;
};

class CDSPResampler16 : public CDSPResampler {
public:
    CDSPResampler16(const double SrcSampleRate, const double DstSampleRate, const int aMaxInLen,
                    const double ReqTransBand = 2.0)
        : CDSPResampler(SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, 136.45, fprLinearPhase) {}
};

class CDSPResampler16IR : public CDSPResampler {
public:
    CDSPResampler16IR(const double SrcSampleRate, const double DstSampleRate, const int aMaxInLen,
                      const double ReqTransBand = 2.0)
        : CDSPResampler(SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, 109.56, fprLinearPhase) {}
};

class CDSPResampler24 : public CDSPResampler {
public:
    CDSPResampler24(const double SrcSampleRate, const double DstSampleRate, const int aMaxInLen,
                    const double ReqTransBand = 2.0)
        : CDSPResampler(SrcSampleRate, DstSampleRate, aMaxInLen, ReqTransBand, 180.15, fprLinearPhase) {}
};

} // namespace r8b

#endif // R8B_CDSPRESAMPLER_B200_INCLUDED

// r8b_format.cuh -- the conversion kernels between caller-side sample buffers and the planar fp64 streams, templated on
// the sample format (semantics: r8b_format.cu).  r8b_format.cu instantiates them for the wide formats, r8b_format_bytes.cu
// for the one-byte formats.
#pragma once
#include "r8b_kernels.h"

#include <climits>

#include "r8b_codec.cuh"
#include "r8b_dither.cuh"

namespace r8bgpu {

template <int FMT>
__device__ __forceinline__ double load_sample(const unsigned char* __restrict__ base, size_t idx)
{
    if (FMT == FMT_F64) return reinterpret_cast<const double*>(base)[idx];
    if (FMT == FMT_F32) return (double) reinterpret_cast<const float*>(base)[idx];
    if (FMT == FMT_S16) return (double) reinterpret_cast<const short*>(base)[idx];
    if (FMT == FMT_S32) return (double) reinterpret_cast<const int*>(base)[idx];
    if (is_byte_format(FMT)) return (double) byte_decode(FMT, base[idx]);
    const unsigned char* p = base + 3 * idx; // packed little-endian 24-bit
    const int v = (int) p[0] | ((int) p[1] << 8) | ((int) (signed char) p[2] << 16);
    return (double) v;
}

__device__ __forceinline__ int trunc_sat(double y, int lo, int hi)
{
    if (!(y == y)) return 0;
    const int v = __double2int_rz(y); // saturates at the int32 limits
    return v < lo ? lo : (v > hi ? hi : v);
}

template <int FMT>
__device__ __forceinline__ void store_sample(unsigned char* __restrict__ base, size_t idx, double y)
{
    if (FMT == FMT_F64) {
        reinterpret_cast<double*>(base)[idx] = y;
    } else if (FMT == FMT_F32) {
        reinterpret_cast<float*>(base)[idx] = __double2float_rn(y);
    } else if (FMT == FMT_S16) {
        reinterpret_cast<short*>(base)[idx] = (short) trunc_sat(y, -32768, 32767);
    } else if (FMT == FMT_S32) {
        reinterpret_cast<int*>(base)[idx] = trunc_sat(y, INT_MIN, INT_MAX);
    } else if (is_byte_format(FMT)) { // the int8 (U8) or int16 (µ-law / A-law) value, then its byte (r8b_codec.cuh)
        long long lo, hi;
        dither_range(FMT, lo, hi);
        base[idx] = byte_encode(FMT, trunc_sat(y, (int) lo, (int) hi));
    } else {
        const int v = trunc_sat(y, -8388608, 8388607);
        unsigned char* p = base + 3 * idx;
        p[0] = (unsigned char) (v & 0xff);
        p[1] = (unsigned char) ((v >> 8) & 0xff);
        p[2] = (unsigned char) ((v >> 16) & 0xff);
    }
}

// Extent of channel c in a ragged conversion, from the records launch_ragged uploads: its block length on the way in
// (the history record: m1 - cur_base), its output count on the way out (the last stage's record: e1 - e0).
template <bool TO_F64>
__device__ __forceinline__ long long cvt_extent(const RaggedRec* __restrict__ rr, int c)
{
    return TO_F64 ? rr[c].m1 - rr[c].cur_base : rr[c].e1 - rr[c].e0;
}

// Planar <-> planar: raw channel c at c*raw_stride samples; fp64 channel c at c*f64_stride doubles.
// RAG: n is the largest extent and channel c stops at its own (cvt_extent).
template <int FMT, bool TO_F64, bool RAG>
__global__ void __launch_bounds__(256) k_cvt_planar(unsigned char* raw, size_t raw_stride, double* f64,
                                                    size_t f64_stride, int n, double scale, const RaggedRec* __restrict__ rr)
{
    const int f = blockIdx.x * 256 + threadIdx.x;
    if (f >= n) return;
    const size_t c = blockIdx.y;
    if constexpr (RAG) {
        if (f >= cvt_extent<TO_F64>(rr, (int) c)) return;
    }
    if (TO_F64)
        f64[c * f64_stride + f] = __dmul_rn(load_sample<FMT>(raw, c * raw_stride + f), scale);
    else
        store_sample<FMT>(raw, c * raw_stride + f, __dmul_rn(f64[c * f64_stride + f], scale));
}

// Interleaved <-> planar through a 32x32 shared-memory transpose: frame f of the raw buffer starts at
// f*raw_stride samples, channel c at +c.  Both sides of the transpose touch consecutive addresses.
// RAG: a cell is valid when its frame is below its own channel's extent.  Lane tx holds the extent of channel c0 + tx; the
// side of the transpose whose channel is c0 + r (r is the same across a warp) takes it from lane r with a shuffle that
// all 32 lanes execute, ahead of the bounds test.
template <int FMT, bool TO_F64, bool RAG>
__global__ void __launch_bounds__(256) k_cvt_interleaved(unsigned char* raw, size_t raw_stride, double* f64,
                                                         size_t f64_stride, int n, int n_ch, double scale,
                                                         const RaggedRec* __restrict__ rr)
{
    __shared__ double tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5; // 32 x 8
    const int f0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    long long ext_tx = 0;
    if constexpr (RAG) ext_tx = c0 + tx < n_ch ? cvt_extent<TO_F64>(rr, c0 + tx) : 0;
    if (TO_F64) {
        for (int r = ty; r < 32; r += 8) { // r: frame within tile, tx: channel
            const int f = f0 + r, c = c0 + tx;
            bool ok = f < n && c < n_ch;
            if constexpr (RAG) ok = ok && f < ext_tx;
            if (ok) tile[r][tx] = __dmul_rn(load_sample<FMT>(raw, (size_t) f * raw_stride + c), scale);
        }
        __syncthreads();
        for (int r = ty; r < 32; r += 8) { // r: channel within tile, tx: frame
            const int f = f0 + tx, c = c0 + r;
            long long ext = 0;
            if constexpr (RAG) ext = __shfl_sync(0xffffffffu, ext_tx, r); // every lane takes part, whatever its bounds
            bool ok = f < n && c < n_ch;
            if constexpr (RAG) ok = ok && f < ext;
            if (ok) f64[(size_t) c * f64_stride + f] = tile[tx][r];
        }
    } else {
        for (int r = ty; r < 32; r += 8) {
            const int f = f0 + tx, c = c0 + r;
            long long ext = 0;
            if constexpr (RAG) ext = __shfl_sync(0xffffffffu, ext_tx, r);
            bool ok = f < n && c < n_ch;
            if constexpr (RAG) ok = ok && f < ext;
            if (ok) tile[tx][r] = __dmul_rn(f64[(size_t) c * f64_stride + f], scale);
        }
        __syncthreads();
        for (int r = ty; r < 32; r += 8) {
            const int f = f0 + r, c = c0 + tx;
            bool ok = f < n && c < n_ch;
            if constexpr (RAG) ok = ok && f < ext_tx;
            if (ok) store_sample<FMT>(raw, (size_t) f * raw_stride + c, tile[r][tx]);
        }
    }
}

// MAP forms (a mixed batch, r8bgpu_batch_create_mixed): channel c's fp64 row is rec[c].row and its extent rec[c].n, so
// the channels of every part -- each with its rows in its own staging block -- convert in one launch.  Same arithmetic as
// the forms above.  They are overloads without the RAG flag, so the lock-step and RAG instantiations keep their code.
template <int FMT, bool TO_F64>
__global__ void __launch_bounds__(256) k_cvt_planar(unsigned char* raw, size_t raw_stride, const MapRec* __restrict__ rec, int n,
                                                    double scale)
{
    const int f = blockIdx.x * 256 + threadIdx.x;
    if (f >= n) return;
    const size_t c = blockIdx.y;
    if (f >= rec[c].n) return;
    double* row = rec[c].row;
    if (TO_F64)
        row[f] = __dmul_rn(load_sample<FMT>(raw, c * raw_stride + f), scale);
    else
        store_sample<FMT>(raw, c * raw_stride + f, __dmul_rn(row[f], scale));
}

// Lane tx holds the extent and the row of channel c0 + tx; the side of the transpose whose channel is c0 + r takes both
// from lane r with shuffles that all 32 lanes execute, ahead of the bounds test (as in the RAG form).
template <int FMT, bool TO_F64>
__global__ void __launch_bounds__(256) k_cvt_interleaved(unsigned char* raw, size_t raw_stride, const MapRec* __restrict__ rec,
                                                         int n, int n_ch, double scale)
{
    __shared__ double tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5; // 32 x 8
    const int f0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    long long ext_tx = 0, row_tx = 0;
    if (c0 + tx < n_ch) {
        ext_tx = rec[c0 + tx].n;
        row_tx = (long long) rec[c0 + tx].row;
    }
    if (TO_F64) {
        for (int r = ty; r < 32; r += 8) { // r: frame within tile, tx: channel
            const int f = f0 + r, c = c0 + tx;
            if (f < n && c < n_ch && f < ext_tx)
                tile[r][tx] = __dmul_rn(load_sample<FMT>(raw, (size_t) f * raw_stride + c), scale);
        }
        __syncthreads();
        for (int r = ty; r < 32; r += 8) { // r: channel within tile, tx: frame
            const int f = f0 + tx, c = c0 + r;
            const long long ext = __shfl_sync(0xffffffffu, ext_tx, r); // every lane takes part, whatever its bounds
            double* row = (double*) __shfl_sync(0xffffffffu, row_tx, r);
            if (f < n && c < n_ch && f < ext) row[f] = tile[tx][r];
        }
    } else {
        for (int r = ty; r < 32; r += 8) {
            const int f = f0 + tx, c = c0 + r;
            const long long ext = __shfl_sync(0xffffffffu, ext_tx, r);
            const double* row = (const double*) __shfl_sync(0xffffffffu, row_tx, r);
            if (f < n && c < n_ch && f < ext) tile[tx][r] = __dmul_rn(row[f], scale);
        }
        __syncthreads();
        for (int r = ty; r < 32; r += 8) {
            const int f = f0 + r, c = c0 + tx;
            if (f < n && c < n_ch && f < ext_tx) store_sample<FMT>(raw, (size_t) f * raw_stride + c, tile[r][tx]);
        }
    }
}

template <int FMT, bool TO_F64>
static void launch_cvt_map_inst(void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch, double scale,
                                cudaStream_t st)
{
    if (interleaved) {
        dim3 grid((unsigned) ((n + 31) / 32), (unsigned) ((n_ch + 31) / 32));
        k_cvt_interleaved<FMT, TO_F64><<<grid, 256, 0, st>>>((unsigned char*) raw, raw_stride, rec, n, n_ch, scale);
    } else {
        dim3 grid((unsigned) ((n + 255) / 256), (unsigned) n_ch);
        k_cvt_planar<FMT, TO_F64><<<grid, 256, 0, st>>>((unsigned char*) raw, raw_stride, rec, n, scale);
    }
}

template <int FMT, bool TO_F64>
static void launch_cvt_inst(void* raw, bool interleaved, size_t raw_stride, double* f64, size_t f64_stride, int n,
                            int n_ch, double scale, cudaStream_t st, const RaggedRec* rr)
{
    if (interleaved) {
        dim3 grid((unsigned) ((n + 31) / 32), (unsigned) ((n_ch + 31) / 32));
        if (rr != nullptr)
            k_cvt_interleaved<FMT, TO_F64, true><<<grid, 256, 0, st>>>((unsigned char*) raw, raw_stride, f64, f64_stride, n,
                                                                      n_ch, scale, rr);
        else
            k_cvt_interleaved<FMT, TO_F64, false><<<grid, 256, 0, st>>>((unsigned char*) raw, raw_stride, f64, f64_stride, n,
                                                                       n_ch, scale, nullptr);
    } else {
        dim3 grid((unsigned) ((n + 255) / 256), (unsigned) n_ch);
        if (rr != nullptr)
            k_cvt_planar<FMT, TO_F64, true><<<grid, 256, 0, st>>>((unsigned char*) raw, raw_stride, f64, f64_stride, n, scale, rr);
        else
            k_cvt_planar<FMT, TO_F64, false><<<grid, 256, 0, st>>>((unsigned char*) raw, raw_stride, f64, f64_stride, n, scale,
                                                                  nullptr);
    }
}

// Dithered integer output.  A warp owns 32 channels (lane = channel) and the frames [blockIdx.x * span, +span) of each,
// moved in [32 channels x 32 frames] tiles through shared memory: the fp64 rows are read with lane = frame (coalesced per
// row), every lane then walks its own channel's 32 frames in order with the error history in registers, and the integers
// go out with lane = frame (planar rows) or lane = channel (interleaved frames), consecutive addresses either way.  The
// history comes from err at the channel's first frame and the last 16 errors of the call go back, at slot m & 15 of the
// channel's m-th dithered output, so a frame range split over CTAs (flat TPDF: no feedback) needs no hand-over.  One
// launch converts either the shaped channels (shaped: one pass over all frames) or the flat ones.
template <int FMT, bool IL>
__global__ void __launch_bounds__(128) k_dither_shape(unsigned char* raw, size_t raw_stride, const DitherRec* __restrict__ rec,
                                                      const DitherCfg* __restrict__ cfg, double* __restrict__ err, int n_ch,
                                                      int span, double scale, bool shaped)
{
    __shared__ double ty[4][32][33]; // fp64 outputs in, each replaced by its quantised value
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    const int cb = (blockIdx.y * 4 + wp) * 32, c = cb + lane;
    if (cb >= n_ch) return; // the whole warp
    long long n = 0, n0 = 0, m0 = 0;
    const double* row = nullptr;
    unsigned long long seed = 0;
    int K = 0;
    if (c < n_ch && cfg[c].kind != R8BGPU_DITHER_OFF && (cfg[c].n_taps > 0) == shaped) {
        n = rec[c].n;
        n0 = rec[c].n0;
        m0 = rec[c].m0;
        row = rec[c].row;
        seed = cfg[c].seed;
        K = cfg[c].n_taps;
    }
    const long long f_lo = (long long) blockIdx.x * span;
    const long long f_hi = f_lo + span < n ? f_lo + span : n; // this lane's frames [f_lo, f_hi)
    double tap[kDitherTaps], eh[kDitherTaps];
#pragma unroll
    for (int k = 0; k < kDitherTaps; k++) {
        tap[k] = k < K ? cfg[c].taps[k] : 0.0;
        eh[k] = k < K && f_lo < f_hi ? err[(size_t) c * kDitherTaps + ((m0 + f_lo - 1 - k) & (kDitherTaps - 1))] : 0.0;
    }
    long long lo, hi;
    dither_range(FMT, lo, hi);
    const int warp_hi = __reduce_max_sync(0xffffffffu, (int) (f_hi > f_lo ? f_hi - f_lo : 0));
    for (int t = 0; t < warp_hi; t += 32) {
        const long long f0 = f_lo + t;
#pragma unroll
        for (int j = 0; j < 32; j++) { // lane = frame, row of channel cb + j: 32 independent loads in flight
            const long long nj = __shfl_sync(0xffffffffu, f_hi, j);
            const double* rj = (const double*) __shfl_sync(0xffffffffu, (long long) row, j);
            if (f0 + lane < nj) ty[wp][j][lane] = rj[f0 + lane];
        }
        __syncwarp();
        for (int j = 0; j < 32; j++) { // lane = channel, frames in order
            const long long f = f0 + j;
            if (f < f_hi) {
                ty[wp][lane][j] = (double) dither_step(tap, K, eh, seed, n0 + f, __dmul_rn(ty[wp][lane][j], scale), lo, hi);
                if (f >= n - kDitherTaps) err[(size_t) c * kDitherTaps + ((m0 + f) & (kDitherTaps - 1))] = eh[0];
            }
        }
        __syncwarp();
        if (IL) {
            for (int j = 0; j < 32; j++)
                if (f0 + j < f_hi) store_sample<FMT>(raw, (size_t) (f0 + j) * raw_stride + c, ty[wp][lane][j]);
        } else {
#pragma unroll
            for (int j = 0; j < 32; j++) {
                const long long nj = __shfl_sync(0xffffffffu, f_hi, j);
                if (f0 + lane < nj) store_sample<FMT>(raw, (size_t) (cb + j) * raw_stride + f0 + lane, ty[wp][j][lane]);
            }
        }
        __syncwarp();
    }
}

template <int FMT>
static void launch_dither_inst(void* raw, bool interleaved, size_t raw_stride, const DitherRec* rec, const DitherCfg* cfg,
                               double* err, int n, int n_ch, double scale, int span, bool shaped, cudaStream_t st)
{
    dim3 grid((unsigned) ((n + span - 1) / span), (unsigned) ((n_ch + 127) / 128));
    if (interleaved)
        k_dither_shape<FMT, true><<<grid, 128, 0, st>>>((unsigned char*) raw, raw_stride, rec, cfg, err, n_ch, span, scale, shaped);
    else
        k_dither_shape<FMT, false><<<grid, 128, 0, st>>>((unsigned char*) raw, raw_stride, rec, cfg, err, n_ch, span, scale, shaped);
}

// r8b_format_bytes.cu: the dispatch of the one-byte formats (U8, µ-law, A-law); false for any other format.
bool launch_cvt_bytes(int fmt, bool to_f64, void* raw, bool interleaved, size_t raw_stride, double* f64, size_t f64_stride, int n,
                      int n_ch, double scale, cudaStream_t st, const RaggedRec* rr);
bool launch_cvt_map_bytes(int fmt, bool to_f64, void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                          double scale, cudaStream_t st);
bool launch_dither_bytes(int fmt, void* raw, bool interleaved, size_t raw_stride, const DitherRec* rec, const DitherCfg* cfg,
                         double* err, int n, int n_ch, double scale, int span, bool shaped, cudaStream_t st);
// r8b_format_dsd.cu: DSD bytes -> fp64 (input only); n counts samples, raw_stride bytes.
bool launch_dsd_to_f64(int fmt, const void* raw, bool interleaved, size_t raw_stride, double* f64, size_t f64_stride, int n, int n_ch,
                       double scale, cudaStream_t st, const RaggedRec* rr);
bool launch_dsd_to_f64_mapped(int fmt, const void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                              double scale, cudaStream_t st);

} // namespace r8bgpu

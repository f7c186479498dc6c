// r8b_format.cu -- caller-side sample formats: interleaved/planar int16, int24 (packed), int32,
// float32, float64  <->  the planar fp64 streams the resampling kernels work on.
//
// Replaces the per-sample conversion loops the reference runs on the CPU around process():
// CDSPResampler::oneshot<Tin,Tout>() "(double) ip[i]" / "(Tout) op[i]" (CDSPResampler.h:592-651) and
// the de-interleaving of WAV frames around bench/r8bfreesrc.cpp:106-137.  Moving narrow formats over
// PCIe and widening them on the device cuts host<->device bytes 2-4x for real audio.
//
// Semantics with scale == 1: exactly the C++ conversions of oneshot() -- widening is exact, narrowing to
// float rounds to nearest, narrowing to an integer type truncates toward zero; values outside the
// integer range (undefined behaviour in the reference) saturate here, NaN becomes 0.
#include "r8b_kernels.h"

#include <climits>

namespace r8bgpu {

__host__ __device__ int format_bytes(int fmt)
{
    switch (fmt) {
    case FMT_F64: return 8;
    case FMT_F32: return 4;
    case FMT_S16: return 2;
    case FMT_S24: return 3;
    case FMT_S32: return 4;
    default: return 0;
    }
}

template <int FMT>
__device__ __forceinline__ double load_sample(const unsigned char* __restrict__ base, size_t idx)
{
    if (FMT == FMT_F64) return reinterpret_cast<const double*>(base)[idx];
    if (FMT == FMT_F32) return (double) reinterpret_cast<const float*>(base)[idx];
    if (FMT == FMT_S16) return (double) reinterpret_cast<const short*>(base)[idx];
    if (FMT == FMT_S32) return (double) reinterpret_cast<const int*>(base)[idx];
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

template <bool TO_F64>
static bool launch_cvt_map(int fmt, void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                           double scale, cudaStream_t st)
{
    if (n <= 0 || n_ch <= 0) return true;
    switch (fmt) {
    case FMT_F64: launch_cvt_map_inst<FMT_F64, TO_F64>(raw, interleaved, raw_stride, rec, n, n_ch, scale, st); break;
    case FMT_F32: launch_cvt_map_inst<FMT_F32, TO_F64>(raw, interleaved, raw_stride, rec, n, n_ch, scale, st); break;
    case FMT_S16: launch_cvt_map_inst<FMT_S16, TO_F64>(raw, interleaved, raw_stride, rec, n, n_ch, scale, st); break;
    case FMT_S24: launch_cvt_map_inst<FMT_S24, TO_F64>(raw, interleaved, raw_stride, rec, n, n_ch, scale, st); break;
    case FMT_S32: launch_cvt_map_inst<FMT_S32, TO_F64>(raw, interleaved, raw_stride, rec, n, n_ch, scale, st); break;
    default: return false;
    }
    return true;
}

bool launch_to_f64_mapped(int fmt, const void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                          double scale, cudaStream_t st)
{
    return launch_cvt_map<true>(fmt, const_cast<void*>(raw), interleaved, raw_stride, rec, n, n_ch, scale, st);
}

bool launch_from_f64_mapped(int fmt, void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                            double scale, cudaStream_t st)
{
    return launch_cvt_map<false>(fmt, raw, interleaved, raw_stride, rec, n, n_ch, scale, st);
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

template <bool TO_F64>
static bool launch_cvt(int fmt, void* raw, bool interleaved, size_t raw_stride, double* f64, size_t f64_stride,
                       int n, int n_ch, double scale, cudaStream_t st, const RaggedRec* rr)
{
    if (n <= 0 || n_ch <= 0) return true;
    switch (fmt) {
    case FMT_F64: launch_cvt_inst<FMT_F64, TO_F64>(raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr); break;
    case FMT_F32: launch_cvt_inst<FMT_F32, TO_F64>(raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr); break;
    case FMT_S16: launch_cvt_inst<FMT_S16, TO_F64>(raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr); break;
    case FMT_S24: launch_cvt_inst<FMT_S24, TO_F64>(raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr); break;
    case FMT_S32: launch_cvt_inst<FMT_S32, TO_F64>(raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr); break;
    default: return false;
    }
    return true;
}

bool launch_to_f64(int fmt, const void* raw, bool interleaved, size_t raw_stride, double* f64, size_t f64_stride,
                   int n, int n_ch, double scale, cudaStream_t st, const RaggedRec* rr)
{
    return launch_cvt<true>(fmt, const_cast<void*>(raw), interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr);
}

bool launch_from_f64(int fmt, void* raw, bool interleaved, size_t raw_stride, const double* f64, size_t f64_stride,
                     int n, int n_ch, double scale, cudaStream_t st, const RaggedRec* rr)
{
    return launch_cvt<false>(fmt, raw, interleaved, raw_stride, const_cast<double*>(f64), f64_stride, n, n_ch, scale, st, rr);
}

} // namespace r8bgpu

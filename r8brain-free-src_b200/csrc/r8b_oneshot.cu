// r8b_oneshot.cu -- long clips on the whole GPU (r8bgpu_batch_oneshot, include/r8bgpu.h "long clips"): the two kernels
// that move each lane's block between its clip and the ragged chain's fp64 staging rows.
//
// A lane runs one time segment of one clip.  Unlike the ragged conversions (k_cvt_*, one row per channel at c * stride),
// the raw side of a lane is its clip, addressed at the absolute sample index of the call's block (gather) or of the kept
// outputs (scatter), so clips of any length and any number of lanes per clip share one launch.  The per-element
// arithmetic is that of the ragged conversions (r8b_format.cuh, r8b_dsd.cuh) and of the flat TPDF quantiser
// (r8b_dither.cuh), so a lane's bytes are the one-channel run's.
#include "r8b_dsd.cuh"
#include "r8b_format.cuh"

namespace r8bgpu {

namespace {

// element index of sample i of a clip: planar rows are contiguous, interleaved frames are `stride` elements apart
__device__ __forceinline__ size_t clip_elem(long long i, bool interleaved, size_t stride)
{
    return interleaved ? (size_t) i * stride : (size_t) i;
}

template <int FMT>
__global__ void __launch_bounds__(256) k_oneshot_gather(const OneshotRec* __restrict__ rec, bool interleaved, size_t stride,
                                                        double scale)
{
    const OneshotRec r = rec[blockIdx.y];
    const long long f = (long long) blockIdx.x * 256 + threadIdx.x;
    if (f >= r.n) return;
    const long long i = r.pos + f;
    double v;
    if constexpr (FMT == FMT_DSD_LSB || FMT == FMT_DSD_MSB)
        v = dsd_value(r.raw[clip_elem(i >> 3, interleaved, stride)], i, FMT == FMT_DSD_MSB, scale);
    else
        v = __dmul_rn(load_sample<FMT>(r.raw, clip_elem(i, interleaved, stride)), scale);
    r.row[f] = v;
}

template <int FMT>
__global__ void __launch_bounds__(256) k_oneshot_scatter(const OneshotRec* __restrict__ rec, bool interleaved, size_t stride,
                                                         double scale)
{
    const OneshotRec r = rec[blockIdx.y];
    const long long f = (long long) blockIdx.x * 256 + threadIdx.x;
    if (f >= r.n) return;
    const double y = r.row != nullptr ? r.row[f] : 0.0; // no row: the silence of a passthrough clip's tail
    unsigned char* raw = const_cast<unsigned char*>(r.raw);
    const size_t e = clip_elem(r.pos + f, interleaved, stride);
    if (FMT != FMT_F64 && FMT != FMT_F32 && r.dither) {
        long long lo, hi;
        dither_range(FMT, lo, hi);
        double eh[kDitherTaps] = {};
        store_sample<FMT>(raw, e, (double) dither_step(nullptr, 0, eh, r.seed, r.n0 + f, __dmul_rn(y, scale), lo, hi));
    } else {
        store_sample<FMT>(raw, e, __dmul_rn(y, scale));
    }
}

dim3 oneshot_grid(long long max_n, int n_lanes) { return dim3((unsigned) ((max_n + 255) / 256), (unsigned) n_lanes); }

} // namespace

bool launch_oneshot_gather(int fmt, bool interleaved, size_t stride, double scale, const OneshotRec* rec, long long max_n,
                           int n_lanes, cudaStream_t st)
{
    if (max_n <= 0 || n_lanes <= 0) return true;
    const dim3 g = oneshot_grid(max_n, n_lanes);
#define R8B_GATHER(F) k_oneshot_gather<F><<<g, 256, 0, st>>>(rec, interleaved, stride, scale)
    switch (fmt) {
    case FMT_F64: R8B_GATHER(FMT_F64); break;
    case FMT_F32: R8B_GATHER(FMT_F32); break;
    case FMT_S16: R8B_GATHER(FMT_S16); break;
    case FMT_S24: R8B_GATHER(FMT_S24); break;
    case FMT_S32: R8B_GATHER(FMT_S32); break;
    case FMT_U8: R8B_GATHER(FMT_U8); break;
    case FMT_ULAW: R8B_GATHER(FMT_ULAW); break;
    case FMT_ALAW: R8B_GATHER(FMT_ALAW); break;
    case FMT_DSD_LSB: R8B_GATHER(FMT_DSD_LSB); break;
    case FMT_DSD_MSB: R8B_GATHER(FMT_DSD_MSB); break;
    default: return false;
    }
#undef R8B_GATHER
    return true;
}

bool launch_oneshot_scatter(int fmt, bool interleaved, size_t stride, double scale, const OneshotRec* rec, long long max_n,
                            int n_lanes, cudaStream_t st)
{
    if (max_n <= 0 || n_lanes <= 0) return true;
    const dim3 g = oneshot_grid(max_n, n_lanes);
#define R8B_SCATTER(F) k_oneshot_scatter<F><<<g, 256, 0, st>>>(rec, interleaved, stride, scale)
    switch (fmt) {
    case FMT_F64: R8B_SCATTER(FMT_F64); break;
    case FMT_F32: R8B_SCATTER(FMT_F32); break;
    case FMT_S16: R8B_SCATTER(FMT_S16); break;
    case FMT_S24: R8B_SCATTER(FMT_S24); break;
    case FMT_S32: R8B_SCATTER(FMT_S32); break;
    case FMT_U8: R8B_SCATTER(FMT_U8); break;
    case FMT_ULAW: R8B_SCATTER(FMT_ULAW); break;
    case FMT_ALAW: R8B_SCATTER(FMT_ALAW); break;
    default: return false;
    }
#undef R8B_SCATTER
    return true;
}

} // namespace r8bgpu

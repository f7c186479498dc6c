// r8b_format.cu -- caller-side sample formats: interleaved/planar int16, int24 (packed), int32,
// float32, float64  <->  the planar fp64 streams the resampling kernels work on (kernels: r8b_format.cuh; the one-byte
// formats U8, µ-law and A-law are instantiated in r8b_format_bytes.cu; the one-bit DSD inputs have kernels of their own in
// r8b_format_dsd.cu).
//
// Replaces the per-sample conversion loops the reference runs on the CPU around process():
// CDSPResampler::oneshot<Tin,Tout>() "(double) ip[i]" / "(Tout) op[i]" (CDSPResampler.h:592-651) and
// the de-interleaving of WAV frames around bench/r8bfreesrc.cpp:106-137.  Moving narrow formats over
// PCIe and widening them on the device cuts host<->device bytes 2-4x for real audio.
//
// Semantics with scale == 1: exactly the C++ conversions of oneshot() -- widening is exact, narrowing to
// float rounds to nearest, narrowing to an integer type truncates toward zero; values outside the
// integer range (undefined behaviour in the reference) saturate here, NaN becomes 0.
#include "r8b_format.cuh"
#include "r8b_dsd.cuh"

namespace r8bgpu {

__host__ __device__ int format_bytes(int fmt)
{
    switch (fmt) {
    case FMT_F64: return 8;
    case FMT_F32: return 4;
    case FMT_S16: return 2;
    case FMT_S24: return 3;
    case FMT_S32: return 4;
    case FMT_U8:
    case FMT_ULAW:
    case FMT_ALAW:
    case FMT_DSD_LSB:
    case FMT_DSD_MSB: return 1;
    default: return 0;
    }
}

FormatElem format_elem(int fmt) { return FormatElem{format_bytes(fmt), is_dsd_format(fmt) ? 8 : 1}; }

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
    default:
        if (is_dsd_format(fmt)) return TO_F64 && launch_dsd_to_f64_mapped(fmt, raw, interleaved, raw_stride, rec, n, n_ch, scale, st);
        return launch_cvt_map_bytes(fmt, TO_F64, raw, interleaved, raw_stride, rec, n, n_ch, scale, st);
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
    default:
        if (is_dsd_format(fmt)) return TO_F64 && launch_dsd_to_f64(fmt, raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr);
        return launch_cvt_bytes(fmt, TO_F64, raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr);
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

bool launch_dither(int fmt, void* raw, bool interleaved, size_t raw_stride, const DitherRec* rec, const DitherCfg* cfg, double* err,
                   int n, int n_ch, double scale, bool shaped, cudaStream_t st)
{
    if (n <= 0 || n_ch <= 0) return true;
    const int span = shaped ? (n + 31) / 32 * 32 : 256;
    switch (fmt) {
    case FMT_S16: launch_dither_inst<FMT_S16>(raw, interleaved, raw_stride, rec, cfg, err, n, n_ch, scale, span, shaped, st); break;
    case FMT_S24: launch_dither_inst<FMT_S24>(raw, interleaved, raw_stride, rec, cfg, err, n, n_ch, scale, span, shaped, st); break;
    case FMT_S32: launch_dither_inst<FMT_S32>(raw, interleaved, raw_stride, rec, cfg, err, n, n_ch, scale, span, shaped, st); break;
    default: return launch_dither_bytes(fmt, raw, interleaved, raw_stride, rec, cfg, err, n, n_ch, scale, span, shaped, st);
    }
    return true;
}

} // namespace r8bgpu

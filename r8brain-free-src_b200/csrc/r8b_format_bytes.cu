// r8b_format_bytes.cu -- the conversion kernels of r8b_format.cuh for the one-byte sample formats: unsigned 8-bit PCM
// (R8BGPU_U8) and G.711 µ-law / A-law (R8BGPU_ULAW / R8BGPU_ALAW), coded by r8b_codec.cuh.  In their own translation unit,
// so the wide formats' kernels in r8b_format.cu compile exactly as they did before these formats existed.
#include "r8b_format.cuh"

namespace r8bgpu {

bool launch_cvt_bytes(int fmt, bool to_f64, void* raw, bool interleaved, size_t raw_stride, double* f64, size_t f64_stride, int n,
                      int n_ch, double scale, cudaStream_t st, const RaggedRec* rr)
{
#define R8B_CVT(F)                                                                                                              \
    (to_f64 ? launch_cvt_inst<F, true>(raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr)                   \
            : launch_cvt_inst<F, false>(raw, interleaved, raw_stride, f64, f64_stride, n, n_ch, scale, st, rr))
    switch (fmt) {
    case FMT_U8: R8B_CVT(FMT_U8); break;
    case FMT_ULAW: R8B_CVT(FMT_ULAW); break;
    case FMT_ALAW: R8B_CVT(FMT_ALAW); break;
    default: return false;
    }
#undef R8B_CVT
    return true;
}

bool launch_cvt_map_bytes(int fmt, bool to_f64, void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                          double scale, cudaStream_t st)
{
#define R8B_CVT(F)                                                                                                              \
    (to_f64 ? launch_cvt_map_inst<F, true>(raw, interleaved, raw_stride, rec, n, n_ch, scale, st)                               \
            : launch_cvt_map_inst<F, false>(raw, interleaved, raw_stride, rec, n, n_ch, scale, st))
    switch (fmt) {
    case FMT_U8: R8B_CVT(FMT_U8); break;
    case FMT_ULAW: R8B_CVT(FMT_ULAW); break;
    case FMT_ALAW: R8B_CVT(FMT_ALAW); break;
    default: return false;
    }
#undef R8B_CVT
    return true;
}

// U8 is dithered as an int8 value, µ-law / A-law as the int16 value they encode (dither_range)
bool launch_dither_bytes(int fmt, void* raw, bool interleaved, size_t raw_stride, const DitherRec* rec, const DitherCfg* cfg,
                         double* err, int n, int n_ch, double scale, int span, bool shaped, cudaStream_t st)
{
    switch (fmt) {
    case FMT_U8: launch_dither_inst<FMT_U8>(raw, interleaved, raw_stride, rec, cfg, err, n, n_ch, scale, span, shaped, st); break;
    case FMT_ULAW: launch_dither_inst<FMT_ULAW>(raw, interleaved, raw_stride, rec, cfg, err, n, n_ch, scale, span, shaped, st); break;
    case FMT_ALAW: launch_dither_inst<FMT_ALAW>(raw, interleaved, raw_stride, rec, cfg, err, n, n_ch, scale, span, shaped, st); break;
    default: return false;
    }
    return true;
}

} // namespace r8bgpu

// r8b_format_dsd.cu -- one-bit DSD input (r8b_dsd.cuh) -> the planar fp64 streams, for every chain whose first kernel does
// not decode the bits itself: ragged and mixed calls, interleaved input, chains that do not start with a half-band
// decimator (2822400 -> 1411200 starts with a BlockConvolver), passthrough plans, and R8BGPU_NO_FORMAT_FUSION.  Input only:
// a one-bit output needs a sigma-delta modulator, a recursion that is sequential per channel.
//
// One thread per output sample: the eight lanes that share a byte read it once through L1, and every warp store is 32
// consecutive doubles.  Interleaved bytes (byte frame f at f*raw_stride, channel c at +c) are first staged through shared
// memory, read with lane = channel, so that both the byte loads and the fp64 row stores touch consecutive addresses.
// Lengths are multiples of 8 (the C-ABI refuses any other), so a channel's extent ends on a byte boundary.
#include "r8b_dsd.cuh"
#include "r8b_format.cuh"

namespace r8bgpu {

// Planar: byte row c at c*raw_stride.  RAG: n is the largest extent and channel c stops at its own (cvt_extent).
template <bool RAG>
__global__ void __launch_bounds__(256) k_dsd_planar(const unsigned char* __restrict__ raw, size_t raw_stride, double* __restrict__ f64,
                                                    size_t f64_stride, long long n, bool msb, double scale,
                                                    const RaggedRec* __restrict__ rr)
{
    const long long i = (long long) blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const size_t c = blockIdx.y;
    if constexpr (RAG) {
        if (i >= cvt_extent<true>(rr, (int) c)) return;
    }
    f64[c * f64_stride + i] = dsd_load(raw + c * raw_stride, i, msb, scale);
}

// MAP form (a mixed batch): channel c's fp64 row is rec[c].row and its extent rec[c].n.
__global__ void __launch_bounds__(256) k_dsd_planar_map(const unsigned char* __restrict__ raw, size_t raw_stride,
                                                        const MapRec* __restrict__ rec, long long n, bool msb, double scale)
{
    const long long i = (long long) blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const size_t c = blockIdx.y;
    if (i >= rec[c].n) return;
    rec[c].row[i] = dsd_load(raw + c * raw_stride, i, msb, scale);
}

// Interleaved: a CTA takes 32 byte frames (256 samples) of 32 channels.  The bytes land in shared memory with lane =
// channel; then each warp writes whole 256-sample runs of its channels' rows with lane = sample.  Channel c's row and
// extent come from row_of / ext_of (plain, RAG or MAP form).
template <typename Row, typename Ext>
__device__ __forceinline__ void dsd_interleaved_tile(const unsigned char* __restrict__ raw, size_t raw_stride, long long n, int n_ch,
                                                     bool msb, double scale, Row row_of, Ext ext_of)
{
    __shared__ unsigned char tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5; // 32 x 8
    const long long f0 = (long long) blockIdx.x * 32;       // first byte frame of the tile
    const int c0 = blockIdx.y * 32;
    const long long nf = n >> 3;
    for (int r = ty; r < 32; r += 8) { // r: byte frame within the tile, tx: channel
        const long long f = f0 + r;
        if (f < nf && c0 + tx < n_ch) tile[tx][r] = raw[(size_t) f * raw_stride + c0 + tx];
    }
    __syncthreads();
    const long long s0 = f0 * 8; // first sample of the tile
    for (int r = ty; r < 32; r += 8) { // r: channel within the tile; the warp's 32 lanes cover 32 samples at a time
        const int c = c0 + r;
        if (c >= n_ch) break;
        const long long ext = ext_of(c) < n ? ext_of(c) : n;
        double* row = row_of(c);
        for (int j = tx; j < 256; j += 32) {
            const long long i = s0 + j;
            if (i < ext) row[i] = dsd_value(tile[r][j >> 3], j, msb, scale);
        }
    }
}

template <bool RAG>
__global__ void __launch_bounds__(256) k_dsd_interleaved(const unsigned char* __restrict__ raw, size_t raw_stride, double* __restrict__ f64,
                                                         size_t f64_stride, long long n, int n_ch, bool msb, double scale,
                                                         const RaggedRec* __restrict__ rr)
{
    dsd_interleaved_tile(raw, raw_stride, n, n_ch, msb, scale, [&](int c) { return f64 + (size_t) c * f64_stride; },
                         [&](int c) { return RAG ? cvt_extent<true>(rr, c) : n; });
}

__global__ void __launch_bounds__(256) k_dsd_interleaved_map(const unsigned char* __restrict__ raw, size_t raw_stride,
                                                             const MapRec* __restrict__ rec, long long n, int n_ch, bool msb,
                                                             double scale)
{
    dsd_interleaved_tile(raw, raw_stride, n, n_ch, msb, scale, [&](int c) { return rec[c].row; },
                         [&](int c) { return rec[c].n; });
}

static dim3 dsd_grid(bool interleaved, int n, int n_ch)
{
    return interleaved ? dim3((unsigned) ((n / 8 + 31) / 32), (unsigned) ((n_ch + 31) / 32))
                       : dim3((unsigned) ((n + 255) / 256), (unsigned) n_ch);
}

bool launch_dsd_to_f64(int fmt, const void* raw, bool interleaved, size_t raw_stride, double* f64, size_t f64_stride, int n, int n_ch,
                       double scale, cudaStream_t st, const RaggedRec* rr)
{
    if (n <= 0 || n_ch <= 0) return true;
    const unsigned char* r = (const unsigned char*) raw;
    const bool msb = fmt == FMT_DSD_MSB;
    const dim3 grid = dsd_grid(interleaved, n, n_ch);
    if (interleaved) {
        if (rr != nullptr) k_dsd_interleaved<true><<<grid, 256, 0, st>>>(r, raw_stride, f64, f64_stride, n, n_ch, msb, scale, rr);
        else k_dsd_interleaved<false><<<grid, 256, 0, st>>>(r, raw_stride, f64, f64_stride, n, n_ch, msb, scale, nullptr);
    } else {
        if (rr != nullptr) k_dsd_planar<true><<<grid, 256, 0, st>>>(r, raw_stride, f64, f64_stride, n, msb, scale, rr);
        else k_dsd_planar<false><<<grid, 256, 0, st>>>(r, raw_stride, f64, f64_stride, n, msb, scale, nullptr);
    }
    return true;
}

bool launch_dsd_to_f64_mapped(int fmt, const void* raw, bool interleaved, size_t raw_stride, const MapRec* rec, int n, int n_ch,
                              double scale, cudaStream_t st)
{
    if (n <= 0 || n_ch <= 0) return true;
    const unsigned char* r = (const unsigned char*) raw;
    const bool msb = fmt == FMT_DSD_MSB;
    const dim3 grid = dsd_grid(interleaved, n, n_ch);
    if (interleaved) k_dsd_interleaved_map<<<grid, 256, 0, st>>>(r, raw_stride, rec, n, n_ch, msb, scale);
    else k_dsd_planar_map<<<grid, 256, 0, st>>>(r, raw_stride, rec, n, msb, scale);
    return true;
}

} // namespace r8bgpu

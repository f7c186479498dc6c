// r8b_dsd_mod.cu -- K8: the one-bit DSD modulator's walk (r8b_dsdmod.cuh) over a call's fp64 outputs.
//
// The recursion is sequential within a channel and independent across channels, so one lane walks one channel.  A CTA
// holds 32 channels: warp 0 is the walker, warps 1-4 keep it fed.  Per tile of kTileBits output bits per channel:
//   - the feeders stage the 32 channels' next samples into shared memory, already converted (step 1 of the recursion:
//     scale, clamp), double-buffered in rows of kTileBits + 1 doubles, an odd pitch, so the walker's 32 lanes reading
//     sample t of their rows hit distinct banks; and they store the bytes of the tile the walker finished before,
//     coalesced: lanes along a row's bytes (planar) or across the channels of a frame (interleaved);
//   - the walker steps its channel through the tile with the state in registers, packs the bits into 32-bit words and
//     leaves them in shared memory.  Tiles that every lane walks whole (all but a call's first and last) run without a
//     branch per sample, so only the recursion's own dependent chain sets the pace.
// One barrier per tile hands both buffers over.  Bit j of a call (j counted from the channel's first held-back bit) is
// held-back bit j for j < pending, else sample j - pending of the row (or silence past the row's count); byte j / 8 of
// the call holds bits 8 (j / 8) .. 8 (j / 8) + 7.
#include "r8b_dsdmod.cuh"

namespace r8bgpu {

constexpr int kTileBits = 128;
constexpr int kPitch = kTileBits + 1;
constexpr int kFeedWarps = 4;
constexpr int kModThreads = 32 * (1 + kFeedWarps);
constexpr int kModSmem = 2 * 32 * kPitch * (int) sizeof(double) + 2 * 32 * (kTileBits / 32) * (int) sizeof(unsigned int);

__global__ void __launch_bounds__(kModThreads) k_dsd_mod(const DsdModRec* __restrict__ rec, DsdModState* __restrict__ state,
                                                         unsigned char* __restrict__ out, size_t stride, int n_ch,
                                                         bool interleaved, bool msb, double scale)
{
    extern __shared__ double smem[];
    double* in_s = smem;                                                          // [2][32][kPitch]
    unsigned int* out_s = reinterpret_cast<unsigned int*>(smem + 2 * 32 * kPitch); // [2][32][kTileBits / 32]
    __shared__ const double* row_s[32];
    __shared__ int n_s[32], z_s[32], pend_s[32], tot_s[32];
    __shared__ int ntiles_s;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ch0 = blockIdx.x * 32;
    if (warp == 0) {
        const int c = ch0 + lane;
        int tot = 0;
        if (c < n_ch) {
            const DsdModRec r = rec[c];
            row_s[lane] = r.row;
            n_s[lane] = r.n;
            z_s[lane] = r.zeros;
            pend_s[lane] = r.pending;
            tot = r.pending + r.n + r.zeros;
        } else {
            row_s[lane] = nullptr;
            n_s[lane] = z_s[lane] = pend_s[lane] = 0;
        }
        tot_s[lane] = tot;
        int m = tot;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) ntiles_s = (m + kTileBits - 1) / kTileBits;
    }
    __syncthreads();
    const int ntiles = ntiles_s;
    const int ft = tid - 32; // feeder thread index, 0 .. 32 * kFeedWarps - 1

    // feeders: the converted samples of tile k into buffer k & 1 (silence past a row's count).  Every load of the tile
    // is issued before the first is used, so the tile costs about one memory latency.
    const double v0 = dsd_mod_input(0.0, scale);
    constexpr int kRows = 32 / kFeedWarps, kPer = kTileBits / 32;
    auto load = [&](int k) {
        double* buf = in_s + (k & 1) * 32 * kPitch;
        double y[kRows][kPer];
#pragma unroll
        for (int r = 0; r < kRows; r++) {
            const int c = warp - 1 + r * kFeedWarps;
            const long long i0 = (long long) k * kTileBits - pend_s[c] + lane;
#pragma unroll
            for (int q = 0; q < kPer; q++) {
                const long long i = i0 + 32 * q;
                y[r][q] = i >= 0 && i < n_s[c] ? __ldg(row_s[c] + i) : 0.0;
            }
        }
#pragma unroll
        for (int r = 0; r < kRows; r++) {
            const int c = warp - 1 + r * kFeedWarps;
            const long long i0 = (long long) k * kTileBits - pend_s[c] + lane;
#pragma unroll
            for (int q = 0; q < kPer; q++) {
                const long long i = i0 + 32 * q;
                if (i >= 0 && i < n_s[c] + z_s[c]) buf[c * kPitch + lane + 32 * q] = i < n_s[c] ? dsd_mod_input(y[r][q], scale) : v0;
            }
        }
    };
    // feeders: the bytes of tile k from word buffer k & 1, nothing past a channel's last whole byte
    auto store = [&](int k) {
        const unsigned int* w = out_s + (k & 1) * 32 * (kTileBits / 32);
        constexpr int kBytes = kTileBits / 8;
        for (int idx = ft; idx < 32 * kBytes; idx += 32 * kFeedWarps) {
            const int c = interleaved ? (idx & 31) : idx / kBytes;
            const int q = interleaved ? idx >> 5 : idx % kBytes;
            const long long byte = (long long) k * kBytes + q;
            if (byte >= (tot_s[c] >> 3)) continue;
            unsigned int v = (w[c * (kTileBits / 32) + (q >> 2)] >> (8 * (q & 3))) & 0xffu;
            if (msb) v = __brev(v) >> 24;
            out[interleaved ? (size_t) byte * stride + (size_t) (ch0 + c) : (size_t) (ch0 + c) * stride + (size_t) byte] =
                (unsigned char) v;
        }
    };

    DsdFilter f{};
    long long ov = 0;
    unsigned int word = 0, last = 0;
    int pend = 0, tot = 0;
    if (warp == 0) {
        pend = pend_s[lane];
        tot = tot_s[lane];
        if (ch0 + lane < n_ch) {
            const DsdModState& s = state[ch0 + lane];
            f = s.f;
            word = s.pbits & ((1u << pend) - 1u);
        }
    } else if (ntiles > 0) {
        load(0);
    }
    __syncthreads();
    for (int k = 0; k < ntiles; k++) {
        if (warp == 0) {
            const double* buf = in_s + (k & 1) * 32 * kPitch + lane * kPitch;
            unsigned int* w = out_s + (k & 1) * 32 * (kTileBits / 32) + lane * (kTileBits / 32);
            const int j0 = k * kTileBits;
            if (__all_sync(0xffffffffu, j0 >= pend && j0 + kTileBits <= tot)) { // (word is 0 here: j0 >= pend)
#pragma unroll 1
                for (int g = 0; g < kTileBits / 32; g++) {
                    unsigned int wd = 0;
#pragma unroll
                    for (int t = 0; t < 32; t++) wd |= (unsigned int) dsd_mod_step(f, buf[32 * g + t], ov) << t;
                    w[g] = wd;
                }
            } else {
#pragma unroll 1
                for (int t = 0; t < kTileBits; t++) {
                    const int j = j0 + t;
                    if (j >= pend && j < tot) {
                        word |= (unsigned int) dsd_mod_step(f, buf[t], ov) << (t & 31);
                        if (j == tot - 1) last = word;
                    }
                    if ((t & 31) == 31) {
                        w[t >> 5] = word;
                        word = 0;
                    }
                }
            }
        } else {
            if (k + 1 < ntiles) load(k + 1);
            if (k > 0) store(k - 1);
        }
        __syncthreads();
    }
    if (warp != 0) {
        if (ntiles > 0) store(ntiles - 1);
        return;
    }
    if (ch0 + lane >= n_ch) return;
    DsdModState& s = state[ch0 + lane];
    s.overloads += ov;
    if (rec[ch0 + lane].clear) { // the call ends the stream (a flush): the modulator restarts, its overloads stay counted
        s.f = DsdFilter{};
        s.pbits = 0;
        s.npend = 0;
        return;
    }
    s.f = f;
    if (tot > pend) s.pbits = (last >> ((tot & 31) & ~7)) & ((1u << (tot & 7)) - 1u);
    s.npend = tot & 7;
}

cudaError_t launch_dsd_mod(const DsdModRec* rec, DsdModState* state, void* out, bool interleaved, size_t stride, bool msb,
                           double scale, int n_ch, cudaStream_t st)
{
    const cudaError_t e = cudaFuncSetAttribute(k_dsd_mod, cudaFuncAttributeMaxDynamicSharedMemorySize, kModSmem);
    if (e != cudaSuccess) return e;
    k_dsd_mod<<<(n_ch + 31) / 32, kModThreads, kModSmem, st>>>(rec, state, static_cast<unsigned char*>(out), stride, n_ch,
                                                                interleaved, msb, scale);
    return cudaGetLastError();
}

} // namespace r8bgpu

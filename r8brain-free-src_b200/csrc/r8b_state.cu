// r8b_state.cu -- moving streams between batches: a channel's ring windows into its state blob and back.
//
// A channel's device state is a set of power-of-two rings indexed by absolute sample index (idx & mask): the input
// history, one ring per stage link, and the 16-slot dither error history.  Its blob (include/r8bgpu.h, "moving
// streams") holds, for each ring, the window [a0, a0 + len) of the stream as fp64 words.  One launch moves every
// segment of every named channel: segments run along the grid's y, windows along x in 1024-word tiles, consecutive
// threads on consecutive words, so ring reads and blob writes are coalesced except where the window wraps the ring.
//
// The blob's checksum is an order-free sum of per-word terms (state_word_term), so each warp adds its share with one
// atomic and the result does not depend on the order the warps finish in.
#include "r8b_kernels.h"

namespace r8bgpu {

namespace {

constexpr int kStateThreads = 256;
constexpr int kStateTile = 4 * kStateThreads; // words per CTA and segment

__device__ inline void add_sum(unsigned long long* sum, unsigned long long part)
{
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((threadIdx.x & 31) == 0 && part != 0) atomicAdd(sum, part);
}

__global__ void __launch_bounds__(kStateThreads) k_state_pack(const StateSeg* __restrict__ segs, int n_segs)
{
    for (int si = blockIdx.y; si < n_segs; si += gridDim.y) {
        const StateSeg s = segs[si];
        unsigned long long part = 0;
        for (long long k = (long long) blockIdx.x * kStateTile + threadIdx.x; k < s.len && k < ((long long) blockIdx.x + 1) * kStateTile;
             k += kStateThreads) {
            const long long a = s.a0 + k;
            const double v = a >= s.lo ? s.ring[a & s.mask] : 0.0;
            s.blob[k] = v;
            part += state_word_term((unsigned long long) __double_as_longlong(v), (unsigned long long) (s.word0 + k));
        }
        if (s.sum != nullptr) add_sum(s.sum, part); // (header words carry their terms in the checksum word already)
    }
}

__global__ void __launch_bounds__(kStateThreads) k_state_unpack(const StateSeg* __restrict__ segs, int n_segs, bool check)
{
    for (int si = blockIdx.y; si < n_segs; si += gridDim.y) {
        const StateSeg s = segs[si];
        const long long k0 = (long long) blockIdx.x * kStateTile, k1 = k0 + kStateTile;
        if (check) {
            unsigned long long part = 0;
            for (long long k = k0 + threadIdx.x; k < s.len && k < k1; k += kStateThreads)
                part += state_word_term((unsigned long long) __double_as_longlong(s.blob[k]), (unsigned long long) (s.word0 + k));
            add_sum(s.sum, part);
            continue;
        }
        // slot r of the row holds the one index a of [n - cap, n) with a & mask == r (n = a0 + len: the samples so far)
        const long long cap = s.mask + 1, base = s.a0 + s.len - cap;
        for (long long r = k0 + threadIdx.x; r < cap && r < k1; r += kStateThreads) {
            const long long a = base + ((r - base) & s.mask);
            s.ring[r] = a >= s.a0 ? s.blob[a - s.a0] : 0.0;
        }
    }
}

dim3 state_grid(long long span, int n_segs)
{
    return dim3((unsigned) ((span + kStateTile - 1) / kStateTile), (unsigned) (n_segs < 65535 ? n_segs : 65535));
}

} // namespace

void launch_state_pack(const StateSeg* segs, int n_segs, long long max_len, cudaStream_t st)
{
    if (n_segs <= 0 || max_len <= 0) return;
    k_state_pack<<<state_grid(max_len, n_segs), kStateThreads, 0, st>>>(segs, n_segs);
}

void launch_state_unpack(const StateSeg* segs, int n_segs, long long max_span, bool check, cudaStream_t st)
{
    if (n_segs <= 0 || max_span <= 0) return;
    k_state_unpack<<<state_grid(max_span, n_segs), kStateThreads, 0, st>>>(segs, n_segs, check);
}

} // namespace r8bgpu

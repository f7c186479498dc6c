// r8b_fft.cuh -- in-shared-memory fp64 complex FFT building blocks for sm_90a.
//
// Replaces (as arithmetic, not as code) the reference's CPU real-FFT back-ends behind
// CDSPRealFFT::forward/inverse (CDSPRealFFT.h:98-170; fft/pffft_double.c, fft/fft4g.h).
//
// Layout: M = R1*16*16 complex points (R1 in {4,8,16}) live in shared memory as double2 with
// one padding element every 16 (pad()), which makes every pass below bank-conflict free for
// 128-bit accesses.  The forward transform is decimation-in-frequency with the twiddle AFTER
// each radix-R butterfly and leaves the spectrum in mixed-radix digit-reversed order
// (slot_of()); the inverse transform is the exact mirror (twiddle BEFORE the butterfly,
// passes in reverse order), so "forward -> pointwise multiply in slot order -> inverse" never
// needs a reordering pass.  Neither direction scales; 1/M is folded into the filter spectrum.
//
// Each thread owns one radix-R butterfly (R complex values in registers); the butterflies
// are radix-2 networks unrolled at compile time with the trivial roots (1, -i, (1-i)/sqrt2 ...)
// special-cased.  Inter-pass twiddles come from a precomputed table tw[k] = exp(-2*pi*i*k/M)
// (host, long double -> double), read through the read-only cache.
#pragma once
#include <cuda_runtime.h>

#include <cmath>

// R8B_HD: the butterflies are plain arithmetic; host builds of them back the CPU emulation of the fused
// kernel that tests/ runs without a GPU (tests/cpp/fused2_emul.cu).
#define R8B_HD __host__ __device__ __forceinline__
#ifdef __CUDA_ARCH__
#define R8B_LDG(p) __ldg(p)
#else
#define R8B_LDG(p) (*(p))
using std::fma;
#endif

namespace r8bgpu {

__host__ __device__ __forceinline__ constexpr int fft_pad(int i) { return i + (i >> 4); }
__host__ __device__ __forceinline__ constexpr int fft_padded_len(int m) { return m + (m >> 4); }

template <int DIR>
R8B_HD double2 cmul(double2 a, double2 w)
{
    // DIR > 0: a*w ; DIR < 0: a*conj(w)
    if (DIR > 0) return make_double2(fma(a.x, w.x, -a.y * w.y), fma(a.x, w.y, a.y * w.x));
    return make_double2(fma(a.x, w.x, a.y * w.y), fma(a.y, w.x, -a.x * w.y));
}

// a * W_R^K, W_R = exp(-DIR * 2*pi*i / R), 0 <= K < R/2 (compile-time).
template <int R, int K, int DIR>
R8B_HD double2 mul_root(double2 a)
{
    constexpr double kH = 0.70710678118654752440; // sqrt(1/2)
    if constexpr (K == 0) {
        return a;
    } else if constexpr (4 * K == R) {
        return DIR > 0 ? make_double2(a.y, -a.x) : make_double2(-a.y, a.x);
    } else if constexpr (8 * K == R) {
        return DIR > 0 ? make_double2(kH * (a.x + a.y), kH * (a.y - a.x))
                       : make_double2(kH * (a.x - a.y), kH * (a.x + a.y));
    } else if constexpr (8 * K == 3 * R) {
        return DIR > 0 ? make_double2(kH * (a.y - a.x), -kH * (a.x + a.y))
                       : make_double2(-kH * (a.x + a.y), kH * (a.x - a.y));
    } else {
        // only R == 16, K in {1,3,5,7} reach this branch
        constexpr double c1 = 0.92387953251128675613; // cos(pi/8)
        constexpr double s1 = 0.38268343236508977173; // sin(pi/8)
        constexpr double c = (16 * K == R * 1) ? c1 : (16 * K == R * 3) ? s1 : (16 * K == R * 5) ? -s1 : -c1;
        constexpr double s = (16 * K == R * 1) ? s1 : (16 * K == R * 3) ? c1 : (16 * K == R * 5) ? c1 : s1;
        // W = (c, -s) forward
        return DIR > 0 ? make_double2(fma(a.x, c, a.y * s), fma(a.y, c, -a.x * s))
                       : make_double2(fma(a.x, c, -a.y * s), fma(a.y, c, a.x * s));
    }
}

template <int N, int DIR, int I>
struct BflyStage {
    static R8B_HD void run(double2* v)
    {
        const double2 a = v[I], b = v[I + N / 2];
        v[I] = make_double2(a.x + b.x, a.y + b.y);
        v[I + N / 2] = mul_root<N, I, DIR>(make_double2(a.x - b.x, a.y - b.y));
        if constexpr (I + 1 < N / 2) BflyStage<N, DIR, I + 1>::run(v);
    }
};

// Radix-2 DIF network on N register values: input natural order, output k at v[bitrev(k)].
template <int N, int DIR>
struct Network {
    static R8B_HD void run(double2* v)
    {
        BflyStage<N, DIR, 0>::run(v);
        if constexpr (N > 2) {
            Network<N / 2, DIR>::run(v);
            Network<N / 2, DIR>::run(v + N / 2);
        }
    }
};

template <int R>
__host__ __device__ __forceinline__ constexpr int bitrev(int q)
{
    int r = 0;
    for (int b = 1, t = R >> 1; t > 0; b <<= 1, t >>= 1)
        if (q & b) r |= t;
    return r;
}

// Butterfly g (0 <= g < M/R) of one DIF pass over all blocks of length NCUR, data in padded smem.  One thread's work
// in fft_pass_forward; host builds run it "thread" after "thread" (tests/cpp/bclarge_emul.cpp).
template <int M, int NCUR, int R>
R8B_HD void fft_bfly_forward(double2* __restrict__ s, const double2* __restrict__ tw, int g)
{
    constexpr int D = NCUR / R;
    constexpr int TWS = M / NCUR;
    const int blk = g / D, r = g % D;
    const int base = blk * NCUR + r;
    double2 v[R];
#pragma unroll
    for (int j = 0; j < R; j++) v[j] = s[fft_pad(base + j * D)];
    Network<R, +1>::run(v);
#pragma unroll
    for (int q = 0; q < R; q++) {
        double2 x = v[bitrev<R>(q)];
        if (D > 1 && q > 0) x = cmul<+1>(x, R8B_LDG(&tw[r * q * TWS]));
        s[fft_pad(base + q * D)] = x;
    }
}

// Mirror of fft_bfly_forward: combines R transformed sub-blocks of length NCUR/R.
template <int M, int NCUR, int R>
R8B_HD void fft_bfly_inverse(double2* __restrict__ s, const double2* __restrict__ tw, int g)
{
    constexpr int D = NCUR / R;
    constexpr int TWS = M / NCUR;
    const int blk = g / D, r = g % D;
    const int base = blk * NCUR + r;
    double2 v[R];
#pragma unroll
    for (int q = 0; q < R; q++) {
        double2 x = s[fft_pad(base + q * D)];
        if (D > 1 && q > 0) x = cmul<-1>(x, R8B_LDG(&tw[r * q * TWS]));
        v[q] = x;
    }
    Network<R, -1>::run(v);
#pragma unroll
    for (int j = 0; j < R; j++) s[fft_pad(base + j * D)] = v[bitrev<R>(j)];
}

#ifdef __CUDACC__ // block-wide passes: device code only
// One DIF pass over all blocks of length NCUR (M/R butterflies), data in padded smem.
template <int M, int NCUR, int R, int NT>
__device__ __forceinline__ void fft_pass_forward(double2* __restrict__ s,
                                                 const double2* __restrict__ tw, int tid)
{
#pragma unroll 1
    for (int g = tid; g < M / R; g += NT) fft_bfly_forward<M, NCUR, R>(s, tw, g);
}

// Mirror of fft_pass_forward: combines R transformed sub-blocks of length NCUR/R.
template <int M, int NCUR, int R, int NT>
__device__ __forceinline__ void fft_pass_inverse(double2* __restrict__ s,
                                                 const double2* __restrict__ tw, int tid)
{
#pragma unroll 1
    for (int g = tid; g < M / R; g += NT) fft_bfly_inverse<M, NCUR, R>(s, tw, g);
}

// Short transforms (M = 64 .. 512): plain radix-2 stages, spectrum in bit-reversed order.  They only serve the
// reference-exact power-of-two decimation of SHORT low-pass kernels, whose tiles must coincide with the reference's own
// small blocks (2 << BlockLenBits, CDSPFIRFilter.h:461); a few thousand points per tile -- throughput is not a concern.
template <int M, int NT, int DIR>
__device__ __forceinline__ void fft_small(double2* s, const double2* tw, int tid)
{
    if (DIR > 0) {
#pragma unroll 1
        for (int len = M; len >= 2; len >>= 1) {
            const int half = len >> 1, step = M / len;
            for (int b = tid; b < M / 2; b += NT) {
                const int blk = b / half, r = b - blk * half;
                const int i0 = blk * len + r, i1 = i0 + half;
                const double2 a = s[fft_pad(i0)], c = s[fft_pad(i1)];
                s[fft_pad(i0)] = make_double2(a.x + c.x, a.y + c.y);
                const double2 d = make_double2(a.x - c.x, a.y - c.y);
                s[fft_pad(i1)] = r == 0 ? d : cmul<+1>(d, __ldg(&tw[r * step]));
            }
            __syncthreads();
        }
    } else {
#pragma unroll 1
        for (int len = 2; len <= M; len <<= 1) {
            const int half = len >> 1, step = M / len;
            for (int b = tid; b < M / 2; b += NT) {
                const int blk = b / half, r = b - blk * half;
                const int i0 = blk * len + r, i1 = i0 + half;
                const double2 a = s[fft_pad(i0)];
                double2 c = s[fft_pad(i1)];
                if (r != 0) c = cmul<-1>(c, __ldg(&tw[r * step]));
                s[fft_pad(i0)] = make_double2(a.x + c.x, a.y + c.y);
                s[fft_pad(i1)] = make_double2(a.x - c.x, a.y - c.y);
            }
            __syncthreads();
        }
    }
}

// Full transforms.  M = R1 * 256.  Callers must __syncthreads() before (data ready) and the
// functions end with a __syncthreads().
template <int M, int NT>
__device__ __forceinline__ void fft_forward(double2* s, const double2* tw, int tid)
{
    if constexpr (M <= 512) {
        fft_small<M, NT, +1>(s, tw, tid);
    } else {
        if constexpr (M == 8192) { // 2 * 16 * 16 * 16
            fft_pass_forward<M, M, 2, NT>(s, tw, tid);
            __syncthreads();
            fft_pass_forward<M, 4096, 16, NT>(s, tw, tid);
            __syncthreads();
        } else {
            constexpr int R1 = M / 256;
            fft_pass_forward<M, M, R1, NT>(s, tw, tid);
            __syncthreads();
        }
        fft_pass_forward<M, 256, 16, NT>(s, tw, tid);
        __syncthreads();
        fft_pass_forward<M, 16, 16, NT>(s, tw, tid);
        __syncthreads();
    }
}

template <int M, int NT>
__device__ __forceinline__ void fft_inverse(double2* s, const double2* tw, int tid)
{
    if constexpr (M <= 512) {
        fft_small<M, NT, -1>(s, tw, tid);
    } else {
        fft_pass_inverse<M, 16, 16, NT>(s, tw, tid);
        __syncthreads();
        fft_pass_inverse<M, 256, 16, NT>(s, tw, tid);
        __syncthreads();
        if constexpr (M == 8192) {
            fft_pass_inverse<M, 4096, 16, NT>(s, tw, tid);
            __syncthreads();
            fft_pass_inverse<M, M, 2, NT>(s, tw, tid);
            __syncthreads();
        } else {
            constexpr int R1 = M / 256;
            fft_pass_inverse<M, M, R1, NT>(s, tw, tid);
            __syncthreads();
        }
    }
}

#endif // __CUDACC__

// Frequency index k (0..M-1) <-> storage slot after fft_forward.
//   k = q1 + R1*(q2 + 16*q3)  ->  slot = q1*256 + q2*16 + q3
//   M = 8192 has one more (radix-2) leading digit: k = q0 + 2*(q1 + 16*(q2 + 16*q3)) -> slot = q0*4096 + q1*256 + q2*16 + q3
template <int M>
__host__ __device__ __forceinline__ constexpr int slot_of(int k)
{
    if constexpr (M <= 512) {
        return bitrev<M>(k); // short radix-2 transforms: plain bit reversal
    } else if constexpr (M == 8192) {
        return (k % 2) * 4096 + ((k / 2) % 16) * 256 + ((k / 32) % 16) * 16 + (k / 512);
    } else {
        constexpr int R1 = M / 256;
        return (k % R1) * 256 + ((k / R1) % 16) * 16 + (k / (R1 * 16));
    }
}
template <int M>
__host__ __device__ __forceinline__ constexpr int freq_of(int slot)
{
    if constexpr (M <= 512) {
        return bitrev<M>(slot);
    } else if constexpr (M == 8192) {
        return (slot / 4096) + 2 * (((slot / 256) % 16) + 16 * (((slot / 16) % 16) + 16 * (slot % 16)));
    } else {
        constexpr int R1 = M / 256;
        return (slot / 256) + R1 * (((slot / 16) % 16) + 16 * (slot % 16));
    }
}

} // namespace r8bgpu

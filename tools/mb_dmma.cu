// tools/mb_dmma.cu -- is the fp64 tensor path (mma.sync f64 = SASS DMMA) worth using for the whole-step
// interpolator, and in which shape?  (1) raw throughput of m8n8k4 (DMMA.8x8x4) and the sm_90 shapes m16n8k4,
// m16n8k8, m16n8k16 (DMMA.16x8x{4,8,16}), (2) the interpolation as a strided-Hankel GEMM out of shared memory in
// the m8n8k4 and the m16n8k16 form.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/mb_dmma tools/mb_dmma.cu
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void dmma16x4(double (&c)[4], const double* a, const double* b)
{
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(b[0]));
}
__device__ __forceinline__ void dmma16x8(double (&c)[4], const double* a, const double* b)
{
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__device__ __forceinline__ void dmma16x16(double (&c)[4], const double* a, const double* b)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
                 "{%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
                   "d"(b[2]), "d"(b[3]));
}

template <int ILP>
__global__ void __launch_bounds__(512) k_dmma_raw(double* out, int iters)
{
    double c[ILP][2];
#pragma unroll
    for (int i = 0; i < ILP; i++) c[i][0] = c[i][1] = 0.0;
    double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) dmma(c[i][0], c[i][1], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++) s += c[i][0] + c[i][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// K = 4, 8 or 16: m16n8k{K}
template <int K, int ILP>
__global__ void __launch_bounds__(512) k_dmma16_raw(double* out, int iters)
{
    double c[ILP][4];
#pragma unroll
    for (int i = 0; i < ILP; i++) c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0.0;
    double a[K / 2], b[K / 4];
#pragma unroll
    for (int i = 0; i < K / 2; i++) a[i] = threadIdx.x * 1e-3 + i;
#pragma unroll
    for (int i = 0; i < K / 4; i++) b[i] = 1.0 + threadIdx.x * 1e-6 + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) {
            if constexpr (K == 4) dmma16x4(c[i], a, b);
            else if constexpr (K == 8) dmma16x8(c[i], a, b);
            else dmma16x16(c[i], a, b);
        }
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// interpolation of one phase group: out[c][r] = sum_s y[c*in_step + o + s] * Bp[s][r], r < 8, s < 32, cycles c in MB blocks of 8.
// Fragment rows take cycles through the fused kernel's map (cycles 4 apart in a half-warp: conflict-free A loads for odd
// in_step); the window base moves by 7 doubles per iteration.
constexpr int YLEN = 8704, NG = 20, SM_TAPS = 32;
__device__ __forceinline__ int cyc(int block, int row) { return 16 * (block >> 1) + 4 * (row & 3) + 2 * (block & 1) + (row >> 2); }
template <int MB>
__global__ void __launch_bounds__(512, 1) k_interp_dmma(double* out, const double* gbank, int iters, int in_step)
{
    extern __shared__ double sm[];
    double* y = sm;
    double* sbank = sm + YLEN;
    for (int i = threadIdx.x; i < YLEN; i += blockDim.x) y[i] = 1e-3 * i;
    for (int i = threadIdx.x; i < NG * SM_TAPS * 8; i += blockDim.x) sbank[i] = gbank[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int arow = lane >> 2, acol = lane & 3;   // A fragment: row = lane/4, col = lane%4
    const int bk = lane & 3, bn = lane >> 2;       // B fragment: k = lane%4, n = lane/4
    double tot = 0.0;
    for (int it = 0; it < iters; it++) {
        const int g = (warp + it) % NG, base = (it * 7) & 511;
        int yo[MB];
#pragma unroll
        for (int m = 0; m < MB; m++) yo[m] = cyc(m, arow) * in_step + base + acol;
        double c[MB][2];
#pragma unroll
        for (int m = 0; m < MB; m++) c[m][0] = c[m][1] = 0.0;
        const double* gb = sbank + g * SM_TAPS * 8 + bk * 8 + bn;
#pragma unroll
        for (int ks = 0; ks < SM_TAPS / 4; ks++) {
            const double b = gb[ks * 32];
#pragma unroll
            for (int m = 0; m < MB; m++) dmma(c[m][0], c[m][1], y[yo[m] + 4 * ks], b);
        }
#pragma unroll
        for (int m = 0; m < MB; m++) tot += c[m][0] + c[m][1];
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = tot;
}

// the same loop as m16n8k16 products: P tiles of 16 cycles (two blocks of 8 stacked), K in steps of 16 taps; the lane's
// four B values of a K16 step are contiguous (two LDS.128)
template <int P>
__global__ void __launch_bounds__(512, 1) k_interp_dmma16(double* out, const double* gbank, int iters, int in_step)
{
    extern __shared__ double sm[];
    double* y = sm;
    double* sbank = sm + YLEN;
    for (int i = threadIdx.x; i < YLEN; i += blockDim.x) y[i] = 1e-3 * i;
    for (int i = threadIdx.x; i < NG * SM_TAPS * 8; i += blockDim.x) sbank[i] = gbank[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int arow = lane >> 2, acol = lane & 3;
    double tot = 0.0;
    for (int it = 0; it < iters; it++) {
        const int g = (warp + it) % NG, base = (it * 7) & 511;
        int yo[P][2];
#pragma unroll
        for (int m = 0; m < P; m++)
#pragma unroll
            for (int hh = 0; hh < 2; hh++) yo[m][hh] = cyc(2 * m + hh, arow) * in_step + base + acol;
        double c[P][4];
#pragma unroll
        for (int m = 0; m < P; m++) c[m][0] = c[m][1] = c[m][2] = c[m][3] = 0.0;
        const double* gb = sbank + g * SM_TAPS * 8 + lane * 4;
#pragma unroll
        for (int ks = 0; ks < SM_TAPS / 16; ks++) {
            const double2 b01 = *reinterpret_cast<const double2*>(gb + ks * 128);
            const double2 b23 = *reinterpret_cast<const double2*>(gb + ks * 128 + 2);
            const double b[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
            for (int m = 0; m < P; m++) {
                double a[8];
#pragma unroll
                for (int i = 0; i < 8; i++) a[i] = y[yo[m][i & 1] + 16 * ks + 4 * (i >> 1)];
                dmma16x16(c[m], a, b);
            }
        }
#pragma unroll
        for (int m = 0; m < P; m++) tot += c[m][0] + c[m][1] + c[m][2] + c[m][3];
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = tot;
}

template <typename F>
float timeit(F f)
{
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    f();
    cudaDeviceSynchronize();
    cudaEventRecord(a);
    f();
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        printf("launch failed: %s\n", cudaGetErrorString(e));
        return 0.0f / 0.0f;
    }
    return ms;
}

int main()
{
    double *out, *gbank;
    int nsm = 0, khz = 0;
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double ghz = khz * 1e-6;
    printf("%s, %d SMs, clock attribute %.3f GHz (clk figures below use it)\n", prop.name, nsm, ghz);
    cudaMalloc(&out, nsm * 1024 * 8);
    cudaMalloc(&gbank, NG * SM_TAPS * 8 * 8);
    cudaMemset(gbank, 0, NG * SM_TAPS * 8 * 8);
    const int iters = 8192;
    for (int nt : {256, 512}) {
        auto tf = [&](float ms, int ilp, int flop) { return (double) flop * ilp * iters * (nt / 32) * nsm / (ms * 1e-3) / 1e12; };
        float m1 = timeit([&] { k_dmma_raw<1><<<nsm, nt>>>(out, iters); });
        float m2 = timeit([&] { k_dmma_raw<2><<<nsm, nt>>>(out, iters); });
        float m4 = timeit([&] { k_dmma_raw<4><<<nsm, nt>>>(out, iters); });
        printf("DMMA m8n8k4   raw, %2d warps/SM: ILP1 %.2f TF  ILP2 %.2f TF  ILP4 %.2f TF\n", nt / 32, tf(m1, 1, 512), tf(m2, 2, 512),
               tf(m4, 4, 512));
        float a1 = timeit([&] { k_dmma16_raw<4, 1><<<nsm, nt>>>(out, iters); });
        float a2 = timeit([&] { k_dmma16_raw<4, 2><<<nsm, nt>>>(out, iters); });
        float a4 = timeit([&] { k_dmma16_raw<4, 4><<<nsm, nt>>>(out, iters); });
        printf("DMMA m16n8k4  raw, %2d warps/SM: ILP1 %.2f TF  ILP2 %.2f TF  ILP4 %.2f TF\n", nt / 32, tf(a1, 1, 1024), tf(a2, 2, 1024),
               tf(a4, 4, 1024));
        float b1 = timeit([&] { k_dmma16_raw<8, 1><<<nsm, nt>>>(out, iters); });
        float b2 = timeit([&] { k_dmma16_raw<8, 2><<<nsm, nt>>>(out, iters); });
        float b4 = timeit([&] { k_dmma16_raw<8, 4><<<nsm, nt>>>(out, iters); });
        printf("DMMA m16n8k8  raw, %2d warps/SM: ILP1 %.2f TF  ILP2 %.2f TF  ILP4 %.2f TF\n", nt / 32, tf(b1, 1, 2048), tf(b2, 2, 2048),
               tf(b4, 4, 2048));
        float c1 = timeit([&] { k_dmma16_raw<16, 1><<<nsm, nt>>>(out, iters); });
        float c2 = timeit([&] { k_dmma16_raw<16, 2><<<nsm, nt>>>(out, iters); });
        float c4 = timeit([&] { k_dmma16_raw<16, 4><<<nsm, nt>>>(out, iters); });
        printf("DMMA m16n8k16 raw, %2d warps/SM: ILP1 %.2f TF  ILP2 %.2f TF  ILP4 %.2f TF\n", nt / 32, tf(c1, 1, 4096), tf(c2, 2, 4096),
               tf(c4, 4, 4096));
    }
    const int smem = (YLEN + NG * SM_TAPS * 8) * 8, it2 = 2000;
    cudaFuncSetAttribute(k_interp_dmma<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_interp_dmma<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_interp_dmma16<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_interp_dmma16<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_interp_dmma16<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    for (int nt : {256, 512}) {
        float a = timeit([&] { k_interp_dmma<6><<<nsm, nt, smem>>>(out, gbank, it2, 147); });
        float b = timeit([&] { k_interp_dmma<3><<<nsm, nt, smem>>>(out, gbank, it2, 147); });
        float c = timeit([&] { k_interp_dmma16<3><<<nsm, nt, smem>>>(out, gbank, it2, 147); });
        float d = timeit([&] { k_interp_dmma16<2><<<nsm, nt, smem>>>(out, gbank, it2, 147); });
        float e = timeit([&] { k_interp_dmma16<1><<<nsm, nt, smem>>>(out, gbank, it2, 147); });
        // one warp-iteration = (cycles) x 8 phases x 32 taps; m8n8k4 MB blocks = 8 MB cycles, m16n8k16 P tiles = 16 P cycles
        auto clk_per_out = [&](float ms, int cycles) { return ms * 1e-3 * ghz * 1e9 / ((double) it2 * (nt / 32) * cycles * 8); };
        printf("interp, %2d warps/SM: m8n8k4 MB=6 %.3f  MB=3 %.3f | m16n8k16 P=3 %.3f  P=2 %.3f  P=1 %.3f clk per output\n",
               nt / 32, clk_per_out(a, 48), clk_per_out(b, 24), clk_per_out(c, 48), clk_per_out(d, 32), clk_per_out(e, 16));
    }
    printf("%s (reference: register-tiled DFMA loop = 18 clk per warp-tap per 768 outputs/32 taps -> %.3f clk per output)\n",
           cudaGetErrorString(cudaGetLastError()), 18.0 * 32 / 768);
    return 0;
}

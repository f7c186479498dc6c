// tools/mb_dmma_order.cu -- in which order do the fp64 mma.sync shapes (m8n8k4 = DMMA.8x8x4; sm_90: m16n8k4, m16n8k8,
// m16n8k16) accumulate their products, and do their fragments sit where the PTX ISA says?  Random fragments, device
// result compared bit for bit with candidate orders evaluated in fp64 on the host.  Fragments (g = lane/4, t = lane%4):
//   A element a_i: row g + 8 (i%2), column t + 4 (i/2)   (m8n8k4: one element, row g, column t)
//   B element b_i: row t + 4 i, column g
//   C element c_i: row g + 8 (i/2), column 2t + i%2
// A wrong layout shows as large differences against every order; a different order as last-bit differences.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/mb_dmma_order tools/mb_dmma_order.cu
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cuda_runtime.h>

template <int M, int K>
__global__ void k(const double* A, const double* B, const double* C, double* D) // A [M][K], B [K][8], C and D [M][8]
{
    const int lane = threadIdx.x, g = lane >> 2, t = lane & 3;
    constexpr int NA = M * K / 32, NB = K / 4, NC = M / 4;
    double a[NA], b[NB], c[NC];
    for (int i = 0; i < NA; i++) a[i] = A[(g + 8 * (i % 2)) * K + t + 4 * (i / 2)];
    if (M == 8) a[0] = A[g * K + t];
    for (int i = 0; i < NB; i++) b[i] = B[(t + 4 * i) * 8 + g];
    for (int i = 0; i < NC; i++) c[i] = C[(g + 8 * (i / 2)) * 8 + 2 * t + i % 2];
    if constexpr (M == 8)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
    else if constexpr (K == 4)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    else if constexpr (K == 8)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                     "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
                       "d"(b[2]), "d"(b[3]));
    for (int i = 0; i < NC; i++) D[(g + 8 * (i / 2)) * 8 + 2 * t + i % 2] = c[i];
}

static double rnd() { return rand() / (double) RAND_MAX - 0.5; }

template <int M, int K>
void run(const char* name)
{
    double ha[M * K], hb[K * 8], hc[M * 8], hd[M * 8], *da, *db, *dc, *dd;
    cudaMalloc(&da, sizeof ha); cudaMalloc(&db, sizeof hb); cudaMalloc(&dc, sizeof hc); cudaMalloc(&dd, sizeof hd);
    int hits[5] = {0, 0, 0, 0, 0}, total = 0;
    double max_rel = 0.0; // largest |device - ascending chain| relative to the sum of |terms|
    srand(7);
    for (int trial = 0; trial < 200; trial++) {
        for (int i = 0; i < M * K; i++) ha[i] = rnd() * exp2((double) (rand() % 20));
        for (int i = 0; i < K * 8; i++) hb[i] = rnd();
        for (int i = 0; i < M * 8; i++) hc[i] = rnd() * 100;
        cudaMemcpy(da, ha, sizeof ha, cudaMemcpyHostToDevice); cudaMemcpy(db, hb, sizeof hb, cudaMemcpyHostToDevice);
        cudaMemcpy(dc, hc, sizeof hc, cudaMemcpyHostToDevice);
        k<M, K><<<1, 32>>>(da, db, dc, dd);
        cudaMemcpy(hd, dd, sizeof hd, cudaMemcpyDeviceToHost);
        for (int r = 0; r < M; r++)
            for (int n = 0; n < 8; n++) {
                double pa[K], pb[K];
                for (int q = 0; q < K; q++) { pa[q] = ha[r * K + q]; pb[q] = hb[q * 8 + n]; }
                const double c = hc[r * 8 + n], got = hd[r * 8 + n];
                double s0 = c; for (int q = 0; q < K; q++) s0 = fma(pa[q], pb[q], s0);              // ascending chain from C
                double s1 = c; for (int q = K - 1; q >= 0; q--) s1 = fma(pa[q], pb[q], s1);         // descending chain
                double s2 = pa[0] * pb[0]; for (int q = 1; q < K; q++) s2 = fma(pa[q], pb[q], s2); s2 += c; // products, then C
                double s3 = c; // K-blocks of 4: each block a chain from 0, added to the running sum
                for (int q0 = 0; q0 < K; q0 += 4) { double bs = pa[q0] * pb[q0]; for (int q = q0 + 1; q < q0 + 4; q++) bs = fma(pa[q], pb[q], bs); s3 += bs; }
                double pr[K]; for (int q = 0; q < K; q++) pr[q] = pa[q] * pb[q]; // pairwise tree of rounded products, then C
                for (int w = 1; w < K; w *= 2) for (int q = 0; q + w < K; q += 2 * w) pr[q] += pr[q + w];
                const double s4 = pr[0] + c;
                hits[0] += memcmp(&s0, &got, 8) == 0; hits[1] += memcmp(&s1, &got, 8) == 0; hits[2] += memcmp(&s2, &got, 8) == 0;
                hits[3] += memcmp(&s3, &got, 8) == 0; hits[4] += memcmp(&s4, &got, 8) == 0;
                double mag = fabs(c); for (int q = 0; q < K; q++) mag += fabs(pa[q] * pb[q]);
                max_rel = fmax(max_rel, fabs(got - s0) / mag);
                total++;
            }
    }
    printf("%-9s of %d results: ascending FMA chain from C %d | descending %d | products then +C %d | K4 blocks %d | pairwise %d"
           " | max |d - ascending| / sum|terms| %.2e\n", name, total, hits[0], hits[1], hits[2], hits[3], hits[4], max_rel);
    cudaFree(da); cudaFree(db); cudaFree(dc); cudaFree(dd);
}

int main()
{
    run<8, 4>("m8n8k4");
    run<16, 4>("m16n8k4");
    run<16, 8>("m16n8k8");
    run<16, 16>("m16n8k16");
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}

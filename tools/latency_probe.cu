// Micro-benchmark: dependent-chain latencies of FP64 ops and of the ICP solve pieces on sm_90a.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o /tmp/latency_probe tools/latency_probe.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "../kiss-icp_b200/csrc/se3.cuh"
using namespace kb;

template <int OP>
__global__ void chain(double *io, long long *cyc, int n) {
    double x = io[threadIdx.x], y = io[32 + threadIdx.x];
    long long t0 = clock64();
    for (int i = 0; i < n; ++i) {
        if (OP == 0) x = x + y;
        if (OP == 1) x = x * y;
        if (OP == 2) x = fma(x, y, y);
        if (OP == 3) x = x / y;
        if (OP == 4) x = sqrt(x) + y;
        if (OP == 5) x = sin(x) + y;
        if (OP == 6) x = floor(x / y) + y;
    }
    long long t1 = clock64();
    io[64 + threadIdx.x] = x;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void solve_pieces(double *io, long long *cyc) {
    double A[36], b[6], dx[6];
    for (int i = 0; i < 36; ++i) A[i] = io[i];
    for (int i = 0; i < 6; ++i) b[i] = io[36 + i];
    long long t0 = clock64();
    ldlt6_solve_fast(A, b, dx);
    long long t1 = clock64();
    SE3 e = se3_exp(dx);
    long long t2 = clock64();
    SE3 T = se3_identity();
    T.q = Q4{io[42], io[43], io[44], io[45]};
    SE3 r = se3_mul(e, T);
    long long t3 = clock64();
    SE3 ef = se3_exp_fast(dx);
    long long t4 = clock64();
    SE3 rf = se3_mul_fast(ef, T);
    long long t5 = clock64();
    io[50] = r.q.x + r.t.x + rf.q.x + rf.t.y;
    cyc[0] = t1 - t0; cyc[1] = t2 - t1; cyc[2] = t3 - t2; cyc[3] = t4 - t3; cyc[4] = t5 - t4;
}
__global__ void mem_lat(const int *chain_idx, long long *cyc, int n, int *sink) {
    int j = 0;
    long long t0 = clock64();
    for (int i = 0; i < n; ++i) j = __ldcg(&chain_idx[j]);
    long long t1 = clock64();
    *sink = j; cyc[0] = t1 - t0;
}
int main() {
    double h[128]; for (int i = 0; i < 128; ++i) h[i] = 1.0 + 1e-3 * i;
    // SPD matrix
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) h[6*i+j] = (i==j ? 10.0 + i : 0.1 * (i + j));
    h[42]=0.01; h[43]=0.02; h[44]=0.03; h[45]=0.9993;
    double *d; long long *c; cudaMalloc(&d, sizeof(h)); cudaMalloc(&c, 64); cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice);
    long long hc[8]; const char *names[] = {"DADD", "DMUL", "DFMA", "DDIV", "DSQRT+DADD", "sin+DADD", "floor(div)+DADD"};
    const int n = 2000;
    for (int threads : {1, 32}) {
        #define RUN(OP) chain<OP><<<1, threads>>>(d, c, n); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost); printf("%-16s threads=%2d : %.1f cycles/op\n", names[OP], threads, (double)hc[0] / n);
        RUN(0) RUN(1) RUN(2) RUN(3) RUN(4) RUN(5) RUN(6)
    }
    for (int rep = 0; rep < 2; ++rep) {
        solve_pieces<<<1, 1>>>(d, c); cudaMemcpy(hc, c, 40, cudaMemcpyDeviceToHost);
        printf("ldlt6_solve_fast %lld | se3_exp %lld  se3_mul %lld | fast: exp %lld mul %lld cycles\n", hc[0], hc[1], hc[2], hc[3], hc[4]);
    }
    // pointer chase through L2 (16 MB footprint, stride 4 KB) and through a small L1/L2-hot buffer
    for (size_t bytes : {size_t(16) << 20, size_t(256) << 20}) {
        size_t cnt = bytes / 4; int *hi = (int*)malloc(bytes); size_t stride = 1024 + 17;
        for (size_t i = 0; i < cnt; ++i) hi[i] = (int)((i + stride) % cnt);
        int *di, *sink; cudaMalloc(&di, bytes); cudaMalloc(&sink, 4); cudaMemcpy(di, hi, bytes, cudaMemcpyHostToDevice);
        for (int rep = 0; rep < 2; ++rep) { mem_lat<<<1,1>>>(di, c, 3000, sink); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost);
            printf("ld.cg chase footprint %zu MB rep %d: %.0f cycles/load\n", bytes >> 20, rep, (double)hc[0] / 3000); }
        cudaFree(di); free(hi);
    }
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0); printf("clock %d kHz\n", clk);
    return 0;
}

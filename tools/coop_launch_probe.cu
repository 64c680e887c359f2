// Micro-benchmark: the gap between back-to-back cooperative launches shaped like k_register_frame (one 512-thread CTA
// per SM, 100 KB of dynamic shared memory, ~100 us each), launched plainly and with Hopper's programmatic dependent
// launch (cudaLaunchAttributeProgrammaticStreamSerialization beside the cooperative attribute), with and without an event
// record between the launches and a griddepcontrol.launch_dependents trigger. Prints the mean time from the last CTA of
// launch k leaving to the first CTA of launch k + 1 entering.
// nvcc -gencode arch=compute_90a,code=sm_90a -O2 -o /tmp/coop_launch_probe tools/coop_launch_probe.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ unsigned long long gt() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
extern __shared__ char sm[];
__global__ void __launch_bounds__(512, 1) k(unsigned long long *st, int i, int trig) {
    unsigned long long t0 = threadIdx.x == 0 ? gt() : 0;
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (threadIdx.x == 0) atomicMin(&st[3 * i], t0);
    unsigned long long t = gt();
    while (gt() - t < 100000) {}
    sm[threadIdx.x] = 1;
    __syncthreads();
    if (trig) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (threadIdx.x == 0) atomicMax(&st[3 * i + 1], gt());
}
int main() {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    size_t smem = 100 * 1024;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaStream_t s; cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    cudaEvent_t ev[64]; for (auto &e : ev) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    unsigned long long *st; cudaMalloc(&st, 3 * 64 * 8);
    const char *names[] = {"coop", "coop+pdl", "coop+pdl+event between", "coop+pdl no trigger"};
    for (int mode = 0; mode < 4; ++mode) {
        unsigned long long init[3 * 64]; for (int i = 0; i < 64; ++i) { init[3*i] = ~0ull; init[3*i+1] = 0; init[3*i+2]=0; }
        cudaMemcpy(st, init, sizeof(init), cudaMemcpyHostToDevice);
        cudaDeviceSynchronize();
        cudaError_t err = cudaSuccess;
        for (int i = 0; i < 40; ++i) {
            int trig = mode != 3;
            void *args[] = {&st, &i, &trig};
            if (mode == 0) err = cudaLaunchCooperativeKernel((void *)k, dim3(sms), dim3(512), args, smem, s);
            else {
                cudaLaunchAttribute at[2];
                at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
                at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[1].val.programmaticStreamSerializationAllowed = 1;
                cudaLaunchConfig_t cfg = {}; cfg.gridDim = dim3(sms); cfg.blockDim = dim3(512); cfg.dynamicSmemBytes = smem; cfg.stream = s; cfg.attrs = at; cfg.numAttrs = 2;
                err = cudaLaunchKernelExC(&cfg, (void *)k, args);
            }
            if (err != cudaSuccess) { printf("%s: launch error %s\n", names[mode], cudaGetErrorString(err)); cudaGetLastError(); break; }
            if (mode == 2) cudaEventRecord(ev[i], s);
        }
        cudaError_t e2 = cudaStreamSynchronize(s);
        unsigned long long h[3 * 64]; cudaMemcpy(h, st, sizeof(h), cudaMemcpyDeviceToHost);
        double gap = 0; int n = 0;
        for (int i = 10; i < 39; ++i) { gap += (double)((long long)(h[3*(i+1)] - h[3*i+1])); ++n; }
        printf("%s: sync %s, mean gap, last CTA of k left -> first CTA of k+1 entered: %.2f us\n", names[mode], cudaGetErrorString(e2), gap / n * 1e-3);
    }
    return 0;
}

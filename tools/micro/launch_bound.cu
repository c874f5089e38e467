// Microbenchmark: how fast can the GPU retire chains of tiny dependent kernels, as a function of the number of
// concurrent streams?  (Is a 58-kernel forward pass launch-bound?)   nvcc -arch=sm_90a -o launch_bound launch_bound.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <vector>

__global__ void tiny(float* p, int work) {
    asm volatile("griddepcontrol.launch_dependents;");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    float v = p[threadIdx.x];
    for (int i = 0; i < work; ++i) v = v * 1.0001f + 0.5f;
    p[threadIdx.x] = v;
}

int main() {
    const int chain = 58, iters = 200;
    for (int pdl = 0; pdl < 2; ++pdl)
        for (int ctas : {1, 132, 264})
            for (int ns : {1, 2, 4, 8}) {
                std::vector<cudaStream_t> s(ns);
                std::vector<cudaGraphExec_t> g(ns);
                std::vector<float*> buf(ns);
                for (int k = 0; k < ns; ++k) {
                    cudaStreamCreateWithFlags(&s[k], cudaStreamNonBlocking);
                    cudaMalloc(&buf[k], 4096);
                    cudaGraph_t graph;
                    cudaStreamBeginCapture(s[k], cudaStreamCaptureModeThreadLocal);
                    for (int i = 0; i < chain; ++i) {
                        cudaLaunchConfig_t cfg = {};
                        cfg.gridDim = dim3(ctas);
                        cfg.blockDim = dim3(128);
                        cfg.stream = s[k];
                        cudaLaunchAttribute a[1];
                        a[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
                        a[0].val.programmaticStreamSerializationAllowed = 1;
                        cfg.attrs = a;
                        cfg.numAttrs = (pdl && i > 0) ? 1 : 0;
                        cudaLaunchKernelEx(&cfg, tiny, buf[k], 200);
                    }
                    cudaStreamEndCapture(s[k], &graph);
                    cudaGraphInstantiate(&g[k], graph, 0);
                    cudaGraphDestroy(graph);
                }
                cudaEvent_t e0, e1;
                cudaEventCreate(&e0);
                cudaEventCreate(&e1);
                for (int k = 0; k < ns; ++k) cudaGraphLaunch(g[k], s[k]);
                cudaDeviceSynchronize();
                cudaEventRecord(e0, s[0]);
                for (int k = 1; k < ns; ++k) cudaStreamWaitEvent(s[k], e0, 0);
                for (int i = 0; i < iters; ++i)
                    for (int k = 0; k < ns; ++k) cudaGraphLaunch(g[k], s[k]);
                std::vector<cudaEvent_t> d(ns);
                for (int k = 1; k < ns; ++k) {
                    cudaEventCreateWithFlags(&d[k], cudaEventDisableTiming);
                    cudaEventRecord(d[k], s[k]);
                    cudaStreamWaitEvent(s[0], d[k], 0);
                }
                cudaEventRecord(e1, s[0]);
                cudaDeviceSynchronize();
                float ms;
                cudaEventElapsedTime(&ms, e0, e1);
                printf("pdl=%d ctas=%3d streams=%d : %.2f us per graph of %d kernels (%.2f us/kernel/stream), aggregate %.2f us/kernel, err=%s\n",
                       pdl, ctas, ns, ms * 1e3 / iters, chain, ms * 1e3 / iters / chain, ms * 1e3 / iters / chain / ns,
                       cudaGetErrorString(cudaGetLastError()));
                for (int k = 0; k < ns; ++k) {
                    cudaGraphExecDestroy(g[k]);
                    cudaStreamDestroy(s[k]);
                    cudaFree(buf[k]);
                }
            }
    return 0;
}

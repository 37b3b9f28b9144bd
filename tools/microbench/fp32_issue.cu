// Microbenchmark: sustained FP32 warp-instruction issue rate per SM on H100 for the instruction forms the FFT
// codelets are made of.  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp32_issue fp32_issue.cu && ./fp32_issue
#include <cstdio>
#include <cuda_runtime.h>

template <int MODE>
__global__ void k(float* out, int iters, float a, float b) {
    float x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) x[i] = threadIdx.x * 0.001f + i;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int rep = 0; rep < 8; ++rep) {
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                if (MODE == 0) x[i] = x[i] + x[(i + 5) & 15];                 // FADD reg,reg (butterfly adds)
                if (MODE == 1) x[i] = fmaf(x[i], a, x[(i + 5) & 15]);         // FFMA reg,reg,reg
                if (MODE == 2) x[i] = fmaf(x[i], 0.99991f, x[(i + 5) & 15]);  // FFMA with an immediate multiplier
                if (MODE == 3) x[i] = x[i] * b;                               // FMUL reg,reg
                if (MODE == 4) x[i] = x[i] * 1.0001f;                         // FMUL immediate
                if (MODE == 5) x[i] = x[i] + 1.5f;                            // FADD immediate
            }
        }
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int MODE>
void run(const char* name) {
    float* out;
    cudaMalloc(&out, 132 * 1024 * sizeof(float));
    const int iters = 2000;
    for (int warps : {4, 8, 16, 32}) {
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        k<MODE><<<132, warps * 32>>>(out, 10, 1.0001f, 0.9999f);
        cudaEventRecord(e0);
        k<MODE><<<132, warps * 32>>>(out, iters, 1.0001f, 0.9999f);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        const double instr = double(iters) * 8 * 16 * warps;  // warp-instructions per SM
        printf("%-28s warps/SM %2d : %.3f warp-instr/clk/SM (at 1.965 GHz)\n", name, warps, instr / (ms * 1e-3 * 1.965e9));
    }
    cudaFree(out);
}

int main() {
    run<0>("FADD r,r");
    run<1>("FFMA r,r,r");
    run<2>("FFMA r,imm,r");
    run<3>("FMUL r,r");
    run<4>("FMUL r,imm");
    run<5>("FADD r,imm");
    return 0;
}

// Microbenchmark: sustained shared-memory data-pipe throughput on H100 for the access patterns of the warp FFT
// (128-bit row reads, 64-bit column writes at row stride 34 float2, pair-interleaved table reads).
#include <cstdio>
#include <cuda_runtime.h>

constexpr int kStride = 34;

template <int MODE>
__global__ void k(float* out, int iters) {
    extern __shared__ float2 sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* tile = sm + warp * (32 * kStride);
    for (int i = lane; i < 32 * kStride; i += 32) tile[i] = make_float2(i, -i);
    __syncwarp();
    float ax = 0.f, ay = 0.f;
    for (int it = 0; it < iters; ++it) {
        if (MODE == 0) {  // 16 x LDS.128, thread reads its row (lane*34 + 2 l): phase-2 pattern
#pragma unroll
            for (int l = 0; l < 16; ++l) {
                const float4 v = *reinterpret_cast<const float4*>(tile + lane * kStride + 2 * l);
                ax += v.x + v.z;
                ay += v.y + v.w;
            }
        } else if (MODE == 1) {  // 32 x STS.64 column writes (k1*34 + lane): phase-1 pattern
#pragma unroll
            for (int k1 = 0; k1 < 32; ++k1) tile[k1 * kStride + lane] = make_float2(ax + k1, ay);
            ax += 1.f;
        } else if (MODE == 2) {  // 16 x LDS.128 table reads, consecutive 16 B per lane
#pragma unroll
            for (int p = 0; p < 16; ++p) {
                const float4 v = *reinterpret_cast<const float4*>(tile + 2 * (p * 32 + lane));
                ax += v.x + v.z;
                ay += v.y + v.w;
            }
        } else {  // the transform's mix per unit: 32 STS.64 + 16 LDS.128 (rows) + 48 LDS.128 (tables) + 8 STS.128
#pragma unroll
            for (int k1 = 0; k1 < 32; ++k1) tile[k1 * kStride + lane] = make_float2(ax + k1, ay);
            __syncwarp();
#pragma unroll
            for (int l = 0; l < 16; ++l) {
                const float4 v = *reinterpret_cast<const float4*>(tile + lane * kStride + 2 * l);
                ax += v.x + v.z;
                ay += v.y + v.w;
            }
#pragma unroll
            for (int p = 0; p < 16; ++p) {
                const float4 v = *reinterpret_cast<const float4*>(tile + 2 * (p * 32 + lane));
                ax += v.x * 0.5f + v.z;
                ay += v.y + v.w * 0.5f;
            }
            __syncwarp();
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = ax + ay;
}

template <int MODE>
void run(const char* name, double wf_per_iter) {
    float* out;
    cudaMalloc(&out, 132 * 1024 * sizeof(float));
    const int iters = 4000;
    for (int warps : {4, 8, 16, 20}) {
        const size_t sm = warps * 32 * kStride * sizeof(float2);
        cudaFuncSetAttribute(k<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        k<MODE><<<132, warps * 32, sm>>>(out, 10);
        cudaEventRecord(e0);
        k<MODE><<<132, warps * 32, sm>>>(out, iters);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        printf("%-34s warps/SM %2d : %.3f wavefronts/clk/SM (128 B each, at 1.965 GHz)\n", name, warps,
               double(iters) * wf_per_iter * warps / (ms * 1e-3 * 1.965e9));
    }
    cudaFree(out);
}

int main() {
    run<0>("LDS.128 row reads (stride 34)", 64);
    run<1>("STS.64 column writes (stride 34)", 64);
    run<2>("LDS.128 table reads", 64);
    run<3>("transform mix (STS.64 + LDS.128)", 64 + 64 + 64);
    return 0;
}

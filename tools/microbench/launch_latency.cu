// Host-to-host overhead of a small CUDA-graph job (what gb200_acquire_grid_host pays around its two kernels), by variant:
//   copy node vs a one-CTA loader kernel reading the pinned (device-mapped) source; cudaStreamSynchronize vs polling a flag the
//   last CTA writes into pinned memory.  Kernels are empty apart from that, so the numbers are pure launch / completion cost.
// build: nvcc -O2 -gencode arch=compute_90a,code=sm_90a -o launch_latency launch_latency.cu
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <vector>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__global__ void k_work(const float4* in, float4* out, int n) {  // touch the data so the copy is a real dependency
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i];
}
__global__ void k_load(const float4* host_mapped, float4* dev, int n) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) dev[i] = host_mapped[i];
}
__global__ void k_tail(const float4* in, float4* host_out, int n, unsigned* counter, volatile unsigned* flag, unsigned seq) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) host_out[i] = in[i];
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0 && flag) {
        if (atomicAdd(counter, 1u) == gridDim.x - 1) {
            *counter = 0;
            __threadfence_system();
            *flag = seq;
        }
    }
}

template <class F>
static double median_us(F fn, int n = 2000) {
    std::vector<double> t;
    for (int k = 0; k < n; ++k) {
        auto a = std::chrono::steady_clock::now();
        fn(k);
        auto b = std::chrono::steady_clock::now();
        t.push_back(std::chrono::duration<double, std::micro>(b - a).count());
    }
    std::sort(t.begin() + n / 10, t.end());
    return t[n / 10 + (n - n / 10) / 2];
}

int main() {
    const int n = 1024;  // float4: 16 KB
    float4 *h_in, *h_out, *d_a, *d_b;
    unsigned *d_counter, *h_flag;
    CK(cudaHostAlloc(&h_in, n * 16, cudaHostAllocMapped));
    CK(cudaHostAlloc(&h_out, 2624 * 16, cudaHostAllocMapped));
    CK(cudaHostAlloc(&h_flag, 64, cudaHostAllocMapped));
    CK(cudaMalloc(&d_a, n * 16));
    CK(cudaMalloc(&d_b, 4096 * 16));
    CK(cudaMalloc(&d_counter, 4));
    CK(cudaMemset(d_counter, 0, 4));
    *h_flag = 0;
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));

    auto capture = [&](int variant, cudaGraphExec_t* exec) -> int {
        cudaGraph_t g;
        CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        if (variant == 0) CK(cudaMemcpyAsync(d_a, h_in, n * 16, cudaMemcpyHostToDevice, st));
        else k_load<<<1, 1024, 0, st>>>(h_in, d_a, n);
        k_work<<<41, 128, 0, st>>>(d_a, d_b, n);
        k_tail<<<128, 384, 0, st>>>(d_b, h_out, 2624, d_counter, nullptr, 0);
        CK(cudaStreamEndCapture(st, &g));
        CK(cudaGraphInstantiate(exec, g, 0));
        cudaGraphDestroy(g);
        return 0;
    };
    cudaGraphExec_t g_copy, g_load;
    if (capture(0, &g_copy) || capture(1, &g_load)) return 1;

    printf("empty kernel + sync                      %.2f us\n", median_us([&](int) { k_work<<<1, 32, 0, st>>>(d_a, d_b, 0); cudaStreamSynchronize(st); }));
    printf("graph{memcpy 16K, k, k->pinned} + sync   %.2f us\n", median_us([&](int) { cudaGraphLaunch(g_copy, st); cudaStreamSynchronize(st); }));
    printf("graph{loader kernel, k, k->pinned} + sync %.2f us\n", median_us([&](int) { cudaGraphLaunch(g_load, st); cudaStreamSynchronize(st); }));
    printf("eager memcpy + 2 kernels + sync          %.2f us\n", median_us([&](int) {
               cudaMemcpyAsync(d_a, h_in, n * 16, cudaMemcpyHostToDevice, st);
               k_work<<<41, 128, 0, st>>>(d_a, d_b, n);
               k_tail<<<128, 384, 0, st>>>(d_b, h_out, 2624, d_counter, nullptr, 0);
               cudaStreamSynchronize(st);
           }));
    printf("eager loader + 2 kernels + sync          %.2f us\n", median_us([&](int) {
               k_load<<<1, 1024, 0, st>>>(h_in, d_a, n);
               k_work<<<41, 128, 0, st>>>(d_a, d_b, n);
               k_tail<<<128, 384, 0, st>>>(d_b, h_out, 2624, d_counter, nullptr, 0);
               cudaStreamSynchronize(st);
           }));
    // flag polling: eager launches (the sequence number is a kernel argument), completion = the flag in pinned memory
    printf("eager loader + 2 kernels + flag poll     %.2f us\n", median_us([&](int k) {
               const unsigned seq = k + 1;
               k_load<<<1, 1024, 0, st>>>(h_in, d_a, n);
               k_work<<<41, 128, 0, st>>>(d_a, d_b, n);
               k_tail<<<128, 384, 0, st>>>(d_b, h_out, 2624, d_counter, h_flag, seq);
               while (*(volatile unsigned*)h_flag != seq) {}
           }));
    cudaStreamSynchronize(st);
    printf("eager memcpy + 2 kernels + flag poll     %.2f us\n", median_us([&](int k) {
               const unsigned seq = 100000 + k;
               cudaMemcpyAsync(d_a, h_in, n * 16, cudaMemcpyHostToDevice, st);
               k_work<<<41, 128, 0, st>>>(d_a, d_b, n);
               k_tail<<<128, 384, 0, st>>>(d_b, h_out, 2624, d_counter, h_flag, seq);
               while (*(volatile unsigned*)h_flag != seq) {}
           }));
    cudaStreamSynchronize(st);
    printf("one kernel reading mapped 16K + flag     %.2f us\n", median_us([&](int k) {
               const unsigned seq = 200000 + k;
               k_tail<<<1, 1024, 0, st>>>(h_in, h_out, 1024, d_counter, h_flag, seq);
               while (*(volatile unsigned*)h_flag != seq) {}
           }));
    cudaStreamSynchronize(st);
    return 0;
}

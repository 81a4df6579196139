// Micro-benchmark (measurement aid, not part of the library): does the residual stream x stay in L2 after the way the proj / fc2
// epilogue updates it (bulk reduce-add performed at L2), so that the LayerNorm pass that follows could read it from there?
// Times lfm::ln_modulate_kernel<8> (M = 16384 rows of 1024 fp32), sweeping the rows upwards and then downwards, right after x was
// (a) written with plain stores, (b) updated with cp.reduce.async.bulk .add.f32 from shared memory (the non-tensor form of the TMA
// reduce the GEMM uses), (c) updated with red.global.add.f32, (d) just read by the same kernel, (e) after a 512 MB flush.
//   mkdir -p build && nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I lfm_b200/csrc tests/tools/l2_residency.cu -o build/l2_residency && build/l2_residency
#include <cstdio>
#include <cuda_runtime.h>
#include "common.cuh"
#include "kernels.cuh"

using namespace lfm;

__global__ void write_plain(float4* x, size_t n4, float v) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) x[i] = make_float4(v, v, v, v);
}
__global__ void update_red(float* x, size_t n, float v) {
    for (size_t i = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) * 4; i < n; i += (size_t)gridDim.x * blockDim.x * 4)
        asm volatile("red.global.add.v4.f32 [%0], {%1, %1, %1, %1};" ::"l"(x + i), "f"(v) : "memory");
}
// each block: 16 KB of shared memory filled once, bulk-reduce-added into consecutive 16 KB pieces of x
__global__ void update_bulk_reduce(float* x, size_t n, float v) {
    __shared__ __align__(128) float buf[4096];
    for (int i = threadIdx.x; i < 4096; i += blockDim.x) buf[i] = v;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0) {
        for (size_t p = (size_t)blockIdx.x * 4096; p < n; p += (size_t)gridDim.x * 4096)
            asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(x + p),
                         "r"((uint32_t)__cvta_generic_to_shared(buf)), "r"(16384u)
                         : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

int main() {
    const int M = 16384, D = 1024;
    const size_t n = (size_t)M * D;
    float *x, *mod, *flush;
    __nv_bfloat16* y;
    cudaMalloc(&x, n * 4);
    cudaMalloc(&y, n * 2);
    cudaMalloc(&mod, 64 * 2 * D * 4);
    cudaMalloc(&flush, 512u << 20);
    cudaMemset(mod, 0, 64 * 2 * D * 4);
    cudaMemset(x, 0, n * 4);
    int dev = 0, sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int smem = ln_smem_bytes(8);
    auto kern = ln_modulate_kernel<8>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    const char* names[] = {"plain stores", "cp.reduce.async.bulk add", "red.global.add.v4.f32", "LayerNorm itself (x just read)", "512 MB flush"};
    for (int down = 0; down < 2; ++down)
        for (int w = 0; w < 5; ++w) {
            float best = 1e9f, sum = 0.f;
            for (int rep = 0; rep < 7; ++rep) {
                cudaMemsetAsync(flush, 1, 512u << 20);
                switch (w) {
                    case 0: write_plain<<<sms * 8, 256>>>(reinterpret_cast<float4*>(x), n / 4, 0.5f); break;
                    case 1: update_bulk_reduce<<<sms * 4, 128>>>(x, n, 0.25f); break;
                    case 2: update_red<<<sms * 8, 256>>>(x, n, 0.25f); break;
                    case 3: kern<<<sms, kLnRows * 32, smem>>>(x, y, mod, mod + D, 2 * D, 256, M, down); break;
                    default: break;
                }
                cudaEventRecord(e0);
                kern<<<sms, kLnRows * 32, smem>>>(x, y, mod, mod + D, 2 * D, 256, M, down);
                cudaEventRecord(e1);
                cudaEventSynchronize(e1);
                float ms;
                cudaEventElapsedTime(&ms, e0, e1);
                if (rep > 0) { best = ms < best ? ms : best; sum += ms; }
            }
            printf("ln_modulate<8> (%-4s) after %-32s: best %.1f us, mean %.1f us\n", down ? "down" : "up", names[w], best * 1e3f, sum / 6 * 1e3f);
        }
    cudaError_t e = cudaDeviceSynchronize();
    printf("status: %s\n", cudaGetErrorString(e));
    return e != cudaSuccess;
}

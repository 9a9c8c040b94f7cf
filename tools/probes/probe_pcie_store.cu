// probe_pcie_store.cu — how fast can SM stores push a scan-sized buffer into mapped pinned host memory, and does the
// store width matter?  (Background: rlca_env_step_host mirrors 8.4 MB of scans per call with 4-byte-per-lane stores,
// i.e. 128 B per warp instruction, and the kernel then drains at ~46 GB/s; the DMA engine reaches ~57 GB/s.)
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o probe_pcie_store probe_pcie_store.cu
#include <cuda_runtime.h>
#include <stdio.h>

template <int W>     // W = floats per lane per store: 1 (128 B / warp), 2 (256 B), 4 (512 B)
__global__ void fill(float *dst, size_t n)
{
    size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * W;
    const size_t stride = (size_t)gridDim.x * blockDim.x * W;
    for (; i + W <= n; i += stride) {
        if (W == 1) dst[i] = (float)i;
        if (W == 2) *reinterpret_cast<float2 *>(dst + i) = make_float2((float)i, 1.f);
        if (W == 4) *reinterpret_cast<float4 *>(dst + i) = make_float4((float)i, 1.f, 2.f, 3.f);
    }
}

template <int W>
static void run(const char *name, float *dst, size_t n, int blocks)
{
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    for (int rep = 0; rep < 3; ++rep) fill<W><<<blocks, 256>>>(dst, n);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    const int iters = 20;
    for (int rep = 0; rep < iters; ++rep) fill<W><<<blocks, 256>>>(dst, n);
    cudaEventRecord(e1);
    cudaDeviceSynchronize();
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    printf("%-28s blocks %5d  %8.1f us  %6.1f GB/s\n", name, blocks, ms / iters * 1e3, n * 4.0 / (ms / iters * 1e-3) / 1e9);
}

int main()
{
    const size_t n = (size_t)4104 * 512;          // one headline scan batch: 8.4 MB
    float *h = nullptr, *d = nullptr, *dev = nullptr;
    cudaHostAlloc(&h, n * 4, cudaHostAllocMapped);
    cudaHostGetDevicePointer(&d, h, 0);
    cudaMalloc(&dev, n * 4);
    for (int blocks : {148, 684, 2052}) {
        run<1>("host, 4 B/lane (128 B/warp)", d, n, blocks);
        run<2>("host, 8 B/lane (256 B/warp)", d, n, blocks);
        run<4>("host, 16 B/lane (512 B/warp)", d, n, blocks);
    }
    run<4>("HBM, 16 B/lane", dev, n, 684);
    // DMA reference
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaMemcpy(h, dev, n * 4, cudaMemcpyDeviceToHost);
    cudaEventRecord(e0);
    for (int rep = 0; rep < 20; ++rep) cudaMemcpyAsync(h, dev, n * 4, cudaMemcpyDeviceToHost);
    cudaEventRecord(e1);
    cudaDeviceSynchronize();
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    printf("%-28s               %8.1f us  %6.1f GB/s\n", "cudaMemcpyAsync D2H", ms / 20 * 1e3, n * 4.0 / (ms / 20 * 1e-3) / 1e9);
    return 0;
}

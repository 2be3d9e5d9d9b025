// Hardware probe: cluster occupancy for the cluster kernel's resource shape, DRAM / L2 bandwidth, device attributes.
// Its occupancy lines are the table the planner in cspn2d_cluster.cu assumes when it plans without a GPU.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/_build/probe tools/probe.cu && tools/_build/probe
#include <cuda_runtime.h>
#include <cstdio>
#include <vector>

__global__ void __launch_bounds__(256, 1) dummy_cluster_kernel(float* p) {
    extern __shared__ float sm[];
    if (p) p[threadIdx.x] = sm[threadIdx.x];
}
__global__ void __launch_bounds__(352, 1) dummy_cluster_kernel352(float* p) {
    extern __shared__ float sm[];
    if (p) p[threadIdx.x] = sm[threadIdx.x];
}

__global__ void read_kernel(const float4* __restrict__ src, size_t n, float* sink, int reps) {
    float acc = 0.f;
    for (int r = 0; r < reps; ++r)
        for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
            float4 v = __ldcg(src + i);
            acc += v.x + v.y + v.z + v.w;
        }
    if (acc == 123.456f) *sink = acc;
}
__global__ void copy_kernel(const float4* __restrict__ src, float4* __restrict__ dst, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = src[i];
}

template <typename K>
void occ(K kern, int threads, int smem, const char* name) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    for (int cs = 1; cs <= 16; ++cs) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(cs * 64);
        cfg.blockDim = dim3(threads);
        cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        int n = -1;
        cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
        printf("occupancy %s threads=%d smem=%d cluster=%2d -> max active clusters %d (%d SMs) %s\n", name, threads, smem, cs, n,
               n * cs, e == cudaSuccess ? "" : cudaGetErrorString(e));
        cudaGetLastError();
    }
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int l2 = 0, smemopt = 0, clk = 0;
    cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, 0);
    cudaDeviceGetAttribute(&smemopt, cudaDevAttrMaxSharedMemoryPerBlockOptin, 0);
    cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("device %s sm_%d%d SMs=%d L2=%d MB smem_optin=%d regs/SM=%d clock=%d kHz mem=%zu MB\n", p.name, p.major, p.minor,
           p.multiProcessorCount, l2 >> 20, smemopt, p.regsPerMultiprocessor, clk, p.totalGlobalMem >> 20);
    occ(dummy_cluster_kernel, 256, 200 * 1024, "k256");
    occ(dummy_cluster_kernel, 256, 100 * 1024, "k256");
    occ(dummy_cluster_kernel352, 352, 200 * 1024, "k352");

    float* sink; cudaMalloc(&sink, 4);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (size_t mb : {16, 32, 48, 64, 96, 128, 256, 1024}) {
        size_t bytes = mb << 20, n = bytes / 16;
        float4 *a, *b; cudaMalloc(&a, bytes); cudaMalloc(&b, bytes);
        cudaMemset(a, 1, bytes);
        int reps = mb <= 128 ? 20 : 4;
        read_kernel<<<p.multiProcessorCount * 8, 512>>>(a, n, sink, 2);
        cudaEventRecord(e0);
        read_kernel<<<p.multiProcessorCount * 8, 512>>>(a, n, sink, reps);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        double rd = (double)bytes * reps / (ms * 1e-3) / 1e9;
        copy_kernel<<<p.multiProcessorCount * 8, 512>>>(a, b, n);
        cudaEventRecord(e0);
        for (int r = 0; r < 5; ++r) copy_kernel<<<p.multiProcessorCount * 8, 512>>>(a, b, n);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        double cp = 2.0 * bytes * 5 / (ms * 1e-3) / 1e9;
        printf("bandwidth working-set %4zu MB: repeated read %.0f GB/s, copy (r+w) %.0f GB/s\n", mb, rd, cp);
        cudaFree(a); cudaFree(b);
    }
    printf("last error: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}

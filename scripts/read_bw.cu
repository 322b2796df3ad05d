// read_bw.cu -- micro-benchmark: achievable HBM READ bandwidth with one persistent CTA per SM for
//   (A) LDG.128 streaming with U loads in flight per thread, (B) cp.async.bulk (TMA) into a smem ring
// of NS slots of SLOT bytes.  Used to size the tensor FIR's input path.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o read_bw read_bw.cu && ./read_bw
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ bool try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok;
}

template <int U>
__global__ void __launch_bounds__(512) ldg_kernel(const float4 *__restrict__ in, size_t n4, float *sink) {
    float acc = 0.f;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + (U - 1) * stride < n4; i += U * stride) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; u++) v[u] = __ldg(in + i + u * stride);
#pragma unroll
        for (int u = 0; u < U; u++) acc += v[u].x + v[u].y + v[u].z + v[u].w;
    }
    if (acc == 123.456f) *sink = acc;
}

// tile-ordered variant: CTA b reads contiguous 64 KiB tiles b, b+grid, ... (the FIR's access pattern)
template <int U>
__global__ void __launch_bounds__(512) ldg_tile_kernel(const float4 *__restrict__ in, size_t n4, float *sink) {
    float acc = 0.f;
    constexpr size_t TILE4 = 65536 / 16;
    const size_t ntiles = n4 / TILE4;
    for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const float4 *p = in + t * TILE4;
        for (int i = threadIdx.x; i + (U - 1) * 512 < (int)TILE4; i += U * 512) {
            float4 v[U];
#pragma unroll
            for (int u = 0; u < U; u++) v[u] = __ldg(p + i + u * 512);
#pragma unroll
            for (int u = 0; u < U; u++) acc += v[u].x + v[u].y + v[u].z + v[u].w;
        }
    }
    if (acc == 123.456f) *sink = acc;
}

template <int SLOT, int NS>
__global__ void __launch_bounds__(64) bulk_kernel(const char *__restrict__ in, size_t bytes, float *sink) {
    extern __shared__ __align__(128) unsigned char sm[];
    __shared__ __align__(8) uint64_t full[NS], empty[NS];
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; i++) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&full[i])));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&empty[i])));
        }
        asm volatile("fence.mbarrier_init.release.cluster;");
    }
    __syncthreads();
    // contiguous 64 KiB tiles round-robin over CTAs, each tile moved as 64K/SLOT bulk copies
    constexpr size_t TILE = 65536;
    const size_t ntiles = bytes / TILE;
    if (threadIdx.x == 0) {                       // producer
        int s = 0; uint32_t ph = 0;
        for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x)
            for (size_t o = 0; o < TILE; o += SLOT) {
                while (!try_wait(smem_u32(&empty[s]), ph ^ 1)) {}
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&full[s])), "r"((uint32_t)SLOT) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_u32(sm + (size_t)s * SLOT)), "l"(in + t * TILE + o), "r"((uint32_t)SLOT), "r"(smem_u32(&full[s])) : "memory");
                if (++s == NS) { s = 0; ph ^= 1; }
            }
    } else if (threadIdx.x == 32) {               // consumer: release immediately
        int s = 0; uint32_t ph = 0; float acc = 0.f;
        for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x)
            for (size_t o = 0; o < TILE; o += SLOT) {
                while (!try_wait(smem_u32(&full[s]), ph)) {}
                acc += reinterpret_cast<float *>(sm + (size_t)s * SLOT)[0];
                asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[s])) : "memory");
                if (++s == NS) { s = 0; ph ^= 1; }
            }
        if (acc == 123.456f) *sink = acc;
    }
}

template <typename F> float time_ms(F f) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    f(); f();
    cudaEventRecord(a);
    for (int i = 0; i < 10; i++) f();
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    return ms / 10;
}

int main() {
    const size_t bytes = (size_t)1 << 30;          // 1 GiB, larger than L2
    char *buf; float *sink;
    cudaMalloc(&buf, bytes); cudaMalloc(&sink, 4);
    cudaMemset(buf, 1, bytes);
    const size_t n4 = bytes / 16;
    auto rep = [&](const char *name, float ms) { printf("%-44s %8.3f ms  %7.1f GB/s\n", name, ms, bytes / ms / 1e6); };
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    for (int g : {sms, 2 * sms, 4 * sms}) {
        char nm[96];
        snprintf(nm, 96, "LDG.128 grid-stride U=4 grid=%d", g); rep(nm, time_ms([&] { ldg_kernel<4><<<g, 512>>>((const float4 *)buf, n4, sink); }));
        snprintf(nm, 96, "LDG.128 grid-stride U=8 grid=%d", g); rep(nm, time_ms([&] { ldg_kernel<8><<<g, 512>>>((const float4 *)buf, n4, sink); }));
    }
    for (int g : {sms, 2 * sms}) {
        char nm[96];
        snprintf(nm, 96, "LDG.128 tile-ordered U=8 grid=%d", g); rep(nm, time_ms([&] { ldg_tile_kernel<8><<<g, 512>>>((const float4 *)buf, n4, sink); }));
    }
#define BULK(SLOT, NS)                                                                                      \
    {                                                                                                       \
        auto k = bulk_kernel<SLOT, NS>;                                                                     \
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SLOT * NS);                    \
        char nm[96]; snprintf(nm, 96, "cp.async.bulk slot=%dK x %d (%dK ring) grid=%d", SLOT / 1024, NS, SLOT * NS / 1024, sms); \
        rep(nm, time_ms([&] { k<<<sms, 64, SLOT * NS>>>(buf, bytes, sink); }));                             \
    }
    BULK(4096, 16) BULK(8192, 8) BULK(8192, 16) BULK(8192, 24) BULK(16384, 4) BULK(16384, 8) BULK(16384, 12) BULK(32768, 4) BULK(32768, 6)
    cudaError_t e = cudaDeviceSynchronize();
    printf("%s\n", cudaGetErrorString(e));
    return 0;
}

// bmma_probe.cu — rate of the binary tensor-core MMA (mma.sync.m16n8k256 .b1 .and.popc) on this GPU.
//
// The column-major evaluator's MMA body (kao_device_t.cuh, kSums == 1) forms its sums with this instruction; its
// cost per candidate is the number of MMAs times the rate measured here.  Two streams per warp:
//   dependent    every MMA accumulates onto the previous one's result: the latency of one MMA
//   independent  kInd accumulators per warp, every warp of a full SM issuing: the throughput of an SM
// Cycles come from clock64() inside the kernel (SM cycles, whatever the clock), wall time from CUDA events.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o bmma_probe tools/bmma_probe.cu && ./bmma_probe
// prints one JSON line.
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ void bmma(int (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2])
{
    asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int kInd>
__global__ void probe(const uint32_t *src, int *out, long long *cycles, int iters)
{
    uint32_t a[4], b[2];
    for (int i = 0; i < 4; ++i) a[i] = src[(threadIdx.x * 4 + i) & 1023];
    for (int i = 0; i < 2; ++i) b[i] = src[(threadIdx.x * 2 + i + 7) & 1023];
    int c[kInd][4] = {};
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int k = 0; k < kInd; ++k) bmma(c[k], a, b);
    }
    __syncthreads();
    const long long t1 = clock64();
    int s = 0;
#pragma unroll
    for (int k = 0; k < kInd; ++k) s += c[k][0] + c[k][1] + c[k][2] + c[k][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int kInd>
static int run(const char *name, int blocks, int threads, int iters, const uint32_t *src, int *out, long long *cyc, bool last)
{
    probe<kInd><<<blocks, threads>>>(src, out, cyc, iters / 16);         // warm-up
    CK(cudaGetLastError());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    probe<kInd><<<blocks, threads>>>(src, out, cyc, iters);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    long long hc[1024];
    CK(cudaMemcpy(hc, cyc, sizeof(long long) * blocks, cudaMemcpyDeviceToHost));
    long long mx = 0;
    for (int i = 0; i < blocks; ++i) mx = hc[i] > mx ? hc[i] : mx;
    const double mmas_per_block = (double)(threads / 32) * iters * kInd;       // warp-level MMAs
    const double cyc_per_mma = (double)mx / mmas_per_block;                    // SM cycles per MMA, one block per SM
    const double ops = 2.0 * 16 * 8 * 256;                                     // AND + POPC-add per MAC
    printf("\"%s\": {\"warps_per_sm\": %d, \"accumulators_per_warp\": %d, \"sm_cycles_per_mma\": %.3f, "
           "\"and_popc_macs_per_clk_per_sm\": %.0f, \"ms\": %.3f, \"tops\": %.1f}%s",
           name, threads / 32, kInd, cyc_per_mma, 16 * 8 * 256 / cyc_per_mma, ms, ops * mmas_per_block * blocks / (ms * 1e-3) / 1e12,
           last ? "" : ", ");
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
    return 0;
}

int main()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    uint32_t *src;
    int *out;
    long long *cyc;
    CK(cudaMalloc(&src, 1024 * sizeof(uint32_t)));
    CK(cudaMemset(src, 0x5A, 1024 * sizeof(uint32_t)));
    CK(cudaMalloc(&out, (size_t)sms * 1024 * sizeof(int)));
    CK(cudaMalloc(&cyc, (size_t)1024 * sizeof(long long)));
    int clk_khz = 0;
    CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
    printf("{\"device\": \"%s\", \"sms\": %d, \"max_sm_clock_mhz\": %d, ", prop.name, sms, clk_khz / 1000);
    // latency: one warp per SM, one accumulator chain
    if (run<1>("dependent", sms, 32, 1 << 16, src, out, cyc, false)) return 1;
    // throughput: 32 warps per SM, 8 independent chains each
    if (run<8>("independent", sms, 1024, 1 << 13, src, out, cyc, false)) return 1;
    // throughput at the evaluator's own shape: 32 warps, 4 n-tile accumulators sharing one A fragment
    if (run<4>("independent_4", sms, 1024, 1 << 14, src, out, cyc, true)) return 1;
    printf("}\n");
    return 0;
}

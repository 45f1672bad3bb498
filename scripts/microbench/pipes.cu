// pipes.cu -- H100 micro-benchmarks that decide the next multiplier formulation (DESIGN.md section 9, item 1).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipes pipes.cu && ./pipes
// Measures, per SM sub-partition, cycles per warp instruction for:
//   (a) IMAD.WIDE.U32 carry chains at ILP 1/2/4/8          -> dependent-issue latency and pipe throughput of the integer multiplier
//   (b) DFMA chains at ILP 1/2/4/8                          -> same for the FP64 pipe
//   (c) IMAD.WIDE and DFMA interleaved                      -> are the two pipes independent (sum of throughputs) or shared?
//   (d) the library's Montgomery multiply (ff.cuh) at 1..16 warps per SM sub-partition -> occupancy needed to saturate the pipe
// Output: one line per experiment; cycles from clock64() around a long unrolled loop, one block per SM.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../../zkevm-circuits_b200/csrc/ff.cuh"

using namespace zkb;

template <int ILP>
__global__ void imad_wide_chain(uint32_t seed, uint64_t *out, long long *cycles, int iters) {
    uint32_t lo[ILP], hi[ILP];
#pragma unroll
    for (int k = 0; k < ILP; ++k) { lo[k] = seed + k + threadIdx.x; hi[k] = seed * 3 + k; }
    const uint32_t a = seed | 1u, b = (seed << 1) | 1u;
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int r = 0; r < 16; ++r) {
#pragma unroll
            for (int k = 0; k < ILP; ++k) {
                // (hi:lo) += a * b with carry chained through the pair: mad.lo.cc / madc.hi  ->  IMAD.WIDE.U32
                asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.u32 %1, %2, %3, %1;" : "+r"(lo[k]), "+r"(hi[k]) : "r"(a), "r"(b));
            }
        }
    }
    const long long t1 = clock64();
    uint64_t acc = 0;
#pragma unroll
    for (int k = 0; k < ILP; ++k) acc += ((uint64_t)hi[k] << 32) | lo[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int ILP>
__global__ void dfma_chain(double seed, double *out, long long *cycles, int iters) {
    double x[ILP];
#pragma unroll
    for (int k = 0; k < ILP; ++k) x[k] = seed + k + threadIdx.x;
    const double a = 1.0000001, b = 1e-9;
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int r = 0; r < 16; ++r) {
#pragma unroll
            for (int k = 0; k < ILP; ++k) x[k] = fma(x[k], a, b);
        }
    }
    const long long t1 = clock64();
    double acc = 0;
#pragma unroll
    for (int k = 0; k < ILP; ++k) acc += x[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

// 4 IMAD.WIDE chains + 4 DFMA chains per thread, interleaved
__global__ void mixed_chain(uint32_t seed, double dseed, uint64_t *out, long long *cycles, int iters) {
    uint32_t lo[4], hi[4];
    double x[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { lo[k] = seed + k + threadIdx.x; hi[k] = seed * 3 + k; x[k] = dseed + k; }
    const uint32_t a = seed | 1u, b = (seed << 1) | 1u;
    const double fa = 1.0000001, fb = 1e-9;
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int r = 0; r < 16; ++r) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.u32 %1, %2, %3, %1;" : "+r"(lo[k]), "+r"(hi[k]) : "r"(a), "r"(b));
                x[k] = fma(x[k], fa, fb);
            }
        }
    }
    const long long t1 = clock64();
    uint64_t acc = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) acc += (((uint64_t)hi[k] << 32) | lo[k]) + (uint64_t)x[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

// the library multiply: each thread squares-and-multiplies a private element; blockDim sets warps per SM
__global__ void montmul_throughput(const Fr *in, Fr *out, long long *cycles, int iters) {
    Fr x = in[threadIdx.x & 31], y = in[(threadIdx.x + 7) & 31];
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < iters; ++i) {
        x = fp_mul(x, y);
        y = fp_mul(y, x);
    }
    const long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = fp_add(x, y);
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

static double avg_cycles(long long *d_cycles, int blocks) {
    long long h[1024];
    cudaMemcpy(h, d_cycles, sizeof(long long) * blocks, cudaMemcpyDeviceToHost);
    double s = 0;
    for (int i = 0; i < blocks; ++i) s += (double)h[i];
    return s / blocks;
}

int main() {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, 0) != cudaSuccess) { printf("no CUDA device\n"); return 1; }
    const int sms = prop.multiProcessorCount, iters = 2000;
    uint64_t *d_out;
    double *d_dout;
    long long *d_cycles;
    Fr *d_fr_in, *d_fr_out;
    cudaMalloc(&d_out, sizeof(uint64_t) * sms * 1024);
    cudaMalloc(&d_dout, sizeof(double) * sms * 1024);
    cudaMalloc(&d_cycles, sizeof(long long) * 1024);
    cudaMalloc(&d_fr_in, sizeof(Fr) * 32);
    cudaMalloc(&d_fr_out, sizeof(Fr) * sms * 1024);
    Fr h_in[32];
    for (int i = 0; i < 32; ++i) h_in[i] = fp_from_u64<FrParams>(1234567ull * (i + 3));
    cudaMemcpy(d_fr_in, h_in, sizeof(h_in), cudaMemcpyHostToDevice);
    printf("device %s, %d SMs\n", prop.name, sms);
    // one warp per sub-partition (128 threads) isolates latency; 4 sub-partitions each run 1 warp
#define RUN_IMAD(ILP) { imad_wide_chain<ILP><<<sms, 128>>>(7, d_out, d_cycles, iters); cudaDeviceSynchronize(); \
        printf("IMAD.WIDE chain  ILP=%d : %.2f cycles per warp-instruction per sub-partition\n", ILP, avg_cycles(d_cycles, sms) / (iters * 16.0 * ILP)); }
    RUN_IMAD(1) RUN_IMAD(2) RUN_IMAD(4) RUN_IMAD(8)
#define RUN_DFMA(ILP) { dfma_chain<ILP><<<sms, 128>>>(1.5, d_dout, d_cycles, iters); cudaDeviceSynchronize(); \
        printf("DFMA chain       ILP=%d : %.2f cycles per warp-instruction per sub-partition\n", ILP, avg_cycles(d_cycles, sms) / (iters * 16.0 * ILP)); }
    RUN_DFMA(1) RUN_DFMA(2) RUN_DFMA(4) RUN_DFMA(8)
    mixed_chain<<<sms, 128>>>(7, 1.5, d_out, d_cycles, iters);
    cudaDeviceSynchronize();
    printf("mixed 4x IMAD.WIDE + 4x DFMA : %.2f cycles per (IMAD.WIDE + DFMA) pair per sub-partition  (independent pipes -> max of the two, shared -> sum)\n",
           avg_cycles(d_cycles, sms) / (iters * 16.0 * 4));
    for (int warps = 1; warps <= 16; warps *= 2) {   // warps per sub-partition
        montmul_throughput<<<sms, 128 * warps>>>(d_fr_in, d_fr_out, d_cycles, 200);
        cudaDeviceSynchronize();
        const double cyc = avg_cycles(d_cycles, sms);
        printf("Montgomery multiply, %2d warp(s)/sub-partition : %.1f cycles per warp-multiply per sub-partition (pipe model: 522)\n", warps,
               cyc / (200.0 * 2 * warps));
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}

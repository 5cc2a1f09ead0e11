// latency_bench.cu -- dependent-issue latencies of one warp on sm_90a (what bounds hqdn3d's lookup chains) and the
// throughput of the fp64 conversion / multiply instructions lapsharp's sharpening expression needs.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o latency_bench tools/latency_bench.cu && ./latency_bench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int N = 4096;

template <int MODE>
__global__ void chain(const int16_t *table, int *out, long long *cyc, int seed)
{
    __shared__ int16_t lut[8192];
    for (int i = threadIdx.x; i < 8192; i += blockDim.x) lut[i] = table[i];
    __syncthreads();
    const char *centre = reinterpret_cast<const char *>(lut + 4096);
    int d = 2 * (seed + (int)threadIdx.x), acc = 0;
    const long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; i++)
    {
        if (MODE == 0)      d = *reinterpret_cast<const int16_t *>(centre + d);                               // LDS -> LDS (table holds even offsets)
        else if (MODE == 1) d = *reinterpret_cast<const int16_t *>(centre + ((d >> 3) & ~1)) + (i & 7);        // LDS, IADD, SHF, LOP
        else if (MODE == 2) { int l = *reinterpret_cast<const int16_t *>(centre + ((d >> 3) & ~1)); int o = l + seed; acc += o; d = o - (i & 15); }   // + a second add
        else if (MODE == 3) d = d + seed;                                                                       // IADD chain (asm keeps it)
        else if (MODE == 4) d = (d >> 3) & ~1;                                                                  // SHF, LOP chain
        else if (MODE == 5) d = d * seed + 1;                                                                   // IMAD chain
        if (MODE == 3 || MODE == 4 || MODE == 5) asm volatile("" : "+r"(d));
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0) cyc[MODE] = t1 - t0;
    out[threadIdx.x] = d + acc;
}

template <int MODE>
__global__ void __launch_bounds__(1024) fp64_rate(int *out, long long *cyc, int seed)
{
    int v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = seed + threadIdx.x + k;
    double dv[8];
#pragma unroll
    for (int k = 0; k < 8; k++) dv[k] = (double)v[k];
    __syncthreads();
    const long long t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < 512; i++)
    {
#pragma unroll
        for (int k = 0; k < 8; k++)
        {
            if (MODE == 0)      { dv[k] = (double)v[k]; v[k] += (int)(__double2hiint(dv[k]) & 1); }    // I2F.F64 (+ a cheap dependency)
            else if (MODE == 1) { dv[k] = __dmul_rn(dv[k], 1.0000001); }                              // DMUL
            else if (MODE == 2) { v[k] = (int)dv[k] + i; dv[k] = __hiloint2double(__double2hiint(dv[k]), v[k]); }   // F2I.F64.TRUNC
            else                { dv[k] = __dadd_rn(dv[k], 1.5); }                                    // DADD
        }
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) cyc[8 + MODE] = t1 - t0;
    int s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s += v[k] + __double2loint(dv[k]);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int main()
{
    int16_t *h = new int16_t[8192];
    for (int i = 0; i < 8192; i++) h[i] = (int16_t)(((i * 37) % 4000 - 2000) & ~1);
    int16_t *dt; int *out; long long *cyc;
    cudaMalloc(&dt, 8192 * 2); cudaMalloc(&out, 1024 * 1024 * 4); cudaMallocManaged(&cyc, 16 * 8);
    cudaMemcpy(dt, h, 8192 * 2, cudaMemcpyHostToDevice);
    for (int rep = 0; rep < 2; rep++)
    {
        chain<0><<<1, 32>>>(dt, out, cyc, 2); chain<1><<<1, 32>>>(dt, out, cyc, 2); chain<2><<<1, 32>>>(dt, out, cyc, 2);
        chain<3><<<1, 32>>>(dt, out, cyc, 2); chain<4><<<1, 32>>>(dt, out, cyc, 2); chain<5><<<1, 32>>>(dt, out, cyc, 3);
        fp64_rate<0><<<132, 1024>>>(out, cyc, 1); fp64_rate<1><<<132, 1024>>>(out, cyc, 1);
        fp64_rate<2><<<132, 1024>>>(out, cyc, 1); fp64_rate<3><<<132, 1024>>>(out, cyc, 1);
        cudaDeviceSynchronize();
    }
    const char *names[6] = { "LDS->LDS", "LDS,IADD,SHF,LOP", "LDS,IADD,IADD,SHF,LOP", "IADD", "SHF,LOP", "IMAD" };
    for (int m = 0; m < 6; m++) printf("chain %-24s %.1f cycles per step\n", names[m], (double)cyc[m] / N);
    const char *fn[4] = { "I2F.F64", "DMUL", "F2I.F64", "DADD" };
    for (int m = 0; m < 4; m++)
        printf("rate  %-24s %.2f lane-ops/clk/SM (1024 threads, 8 independent per thread)\n", fn[m], 1024.0 * 8 * 512 / (double)cyc[8 + m]);
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}

// tools/microbench.cu -- per-SM issue throughput of the instructions the NLMeans
// kernel is built from, measured with clock64 inside one 1024-thread CTA per SM.
// Not part of the product; its numbers justify the instruction mix in DESIGN.md.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define ITER 2048
#define NCH 8   // independent chains per thread

template <int OP>
__device__ __forceinline__ void body(uint32_t (&r)[NCH], uint32_t k0, uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane);

#define DEF_OP32(ID, ASM)                                                                     \
    template <> __device__ __forceinline__ void body<ID>(uint32_t (&r)[NCH], uint32_t k0,     \
        uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane) {                               \
        _Pragma("unroll") for (int i = 0; i < NCH; i++) asm volatile(ASM : "+r"(r[i]) : "r"(k0), "r"(k1)); }
#define DEF_OP64(ID, ASM)                                                                     \
    template <> __device__ __forceinline__ void body<ID>(uint32_t (&r)[NCH], uint32_t k0,     \
        uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane) {                               \
        uint64_t kk = ((uint64_t)k1 << 32) | k0;                                              \
        _Pragma("unroll") for (int i = 0; i < NCH; i++) asm volatile(ASM : "+l"(q[i]) : "l"(kk)); }

DEF_OP32(0,  "add.rn.f32 %0, %0, %1;")
DEF_OP32(1,  "mul.rn.f32 %0, %0, %1;")
DEF_OP32(2,  "fma.rn.f32 %0, %0, %1, %2;")
DEF_OP32(6,  "add.u32 %0, %0, %1;")
DEF_OP32(7,  "mad.lo.u32 %0, %0, %1, %2;")
DEF_OP32(8,  "lop3.b32 %0, %0, %1, %2, 0x96;")
DEF_OP32(9,  "prmt.b32 %0, %0, %1, 0x4321;")
DEF_OP32(10, "min.f32 %0, %0, %1;")
DEF_OP32(11, "cvt.rn.f32.s32 %0, %0;")
DEF_OP32(12, "cvt.rzi.s32.f32 %0, %0;")
DEF_OP32(13, "dp4a.u32.u32 %0, %0, %1, %2;")
DEF_OP32(14, "vabsdiff4.u32.u32.u32.add %0, %0, %1, %2;")
DEF_OP32(15, "add.rz.f32 %0, %0, %1;")
DEF_OP32(16, "mul.rn.sat.f32 %0, %0, %1;")
DEF_OP32(17, "{ .reg .pred p; setp.lt.f32 p, %0, %1; selp.b32 %0, %1, %2, p; }")
DEF_OP32(18, "shf.l.wrap.b32 %0, %0, %1, %2;")
DEF_OP32(19, "{ .reg .b32 t; shl.b32 t, %0, 7; add.u32 %0, t, %1; }")      // LEA candidate
DEF_OP32(20, "cvt.rn.f32.u8 %0, %0;")                                       // I2F.U8
DEF_OP32(21, "sub.u32 %0, %0, %1; add.u32 %0, %0, %2;")                    // IADD3 candidate (2 ptx)
DEF_OP64(22, "add.rn.f64 %0, %0, %1;")
DEF_OP32(23, "shfl.sync.bfly.b32 %0, %0, 1, 0x1f, 0xffffffff;")
// mixes
DEF_OP32(24, "add.rn.f32 %0, %0, %1; add.u32 %0, %0, %2;")                 // FADD + IADD interleaved
DEF_OP32(25, "fma.rn.f32 %0, %0, %1, %2; lop3.b32 %0, %0, %1, %2, 0x96;")  // FFMA + LOP3
DEF_OP32(26, "fma.rn.f32 %0, %0, %1, %2; mad.lo.u32 %0, %0, %1, %2;")      // FFMA + IMAD
DEF_OP32(27, "add.rn.f32 %0, %0, %1; prmt.b32 %0, %0, %1, 0x4321;")        // FADD + PRMT


// independent mixes: the first half of the chains runs op A, the second half op B (no dependency between them) --
// which pairs overlap says which pipe each instruction sits on
#define DEF_MIX32(ID, ASMA, ASMB)                                                             \
    template <> __device__ __forceinline__ void body<ID>(uint32_t (&r)[NCH], uint32_t k0,     \
        uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane) {                               \
        _Pragma("unroll") for (int i = 0; i < NCH / 2; i++) {                                 \
            asm volatile(ASMA : "+r"(r[i]) : "r"(k0), "r"(k1));                               \
            asm volatile(ASMB : "+r"(r[i + NCH / 2]) : "r"(k0), "r"(k1)); } }
#define A_FFMA  "fma.rn.f32 %0, %0, %1, %2;"
#define A_LOP3  "lop3.b32 %0, %0, %1, %2, 0x96;"
#define A_DP4A  "dp4a.u32.u32 %0, %0, %1, %2;"
#define A_VABS  "vabsdiff4.u32.u32.u32.add %0, %0, %1, %2;"
#define A_IADD3 "{ .reg .b32 t; add.u32 t, %0, %1; add.u32 %0, t, %2; }"
#define A_PRMT  "prmt.b32 %0, %0, %1, 0x4321;"
#define A_IMAD  "mad.lo.u32 %0, %0, %1, %2;"
#define A_SHF   "shf.l.wrap.b32 %0, %0, %1, %2;"
DEF_MIX32(44, A_DP4A, A_LOP3)
DEF_MIX32(45, A_DP4A, A_FFMA)
DEF_MIX32(46, A_VABS, A_DP4A)
DEF_MIX32(47, A_VABS, A_LOP3)
DEF_MIX32(48, A_VABS, A_FFMA)
DEF_MIX32(49, A_IADD3, A_FFMA)
DEF_MIX32(50, A_IADD3, A_LOP3)
DEF_MIX32(51, A_IADD3, A_DP4A)
DEF_MIX32(52, A_PRMT, A_LOP3)
DEF_MIX32(53, A_IMAD, A_DP4A)
DEF_MIX32(54, A_SHF, A_LOP3)
DEF_MIX32(55, A_SHF, A_FFMA)
DEF_MIX32(56, A_FFMA, A_LOP3)
DEF_MIX32(57, A_IADD3, A_IADD3)

// shared-memory ops: address chain-free (address from lane), value accumulates
template <> __device__ __forceinline__ void body<30>(uint32_t (&r)[NCH], uint32_t k0, uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane) {
    #pragma unroll
    for (int i = 0; i < NCH; i++) { uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(sm) + (uint32_t)(lane * 4 + i * 128))); r[i] ^= v; }
}
template <> __device__ __forceinline__ void body<31>(uint32_t (&r)[NCH], uint32_t k0, uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane) {
    #pragma unroll
    for (int i = 0; i < NCH; i++) { uint32_t a, b, c, d; asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"((uint32_t)__cvta_generic_to_shared(sm) + (uint32_t)(lane * 16 + i * 512))); r[i] ^= a ^ b ^ c ^ d; }
}
// data-dependent LDS (LUT style): index from register, replicated LUT -> conflict-free
template <> __device__ __forceinline__ void body<32>(uint32_t (&r)[NCH], uint32_t k0, uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane) {
    #pragma unroll
    for (int i = 0; i < NCH; i++) { uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(sm) + ((r[i] & 127u) * 128u + (uint32_t)lane * 4u))); r[i] = v; }
}
// data-dependent LDS, non-replicated 128-entry LUT (random bank conflicts)
template <> __device__ __forceinline__ void body<33>(uint32_t (&r)[NCH], uint32_t k0, uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane) {
    #pragma unroll
    for (int i = 0; i < NCH; i++) { uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(sm) + ((r[i] & 127u) * 4u))); r[i] = v * 2654435761u + lane; }
}
// LDS.64 + STS.64 read-modify-write (accumulator traffic)
template <> __device__ __forceinline__ void body<34>(uint32_t (&r)[NCH], uint32_t k0, uint32_t k1, uint64_t (&q)[NCH], float *sm, int lane) {
    #pragma unroll
    for (int i = 0; i < NCH; i++) { uint32_t a, b; uint32_t ad = (uint32_t)__cvta_generic_to_shared(sm) + (uint32_t)(lane * 8 + i * 256);
        asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "r"(ad)); a += r[i]; b ^= k0;
        asm volatile("st.shared.v2.b32 [%0], {%1,%2};" :: "r"(ad), "r"(a), "r"(b) : "memory"); }
}

template <int OP>
__global__ void __launch_bounds__(1024, 1) bench(uint32_t *out, long long *cycles, uint32_t k0, uint32_t k1)
{
    extern __shared__ float sm[];
    for (int i = threadIdx.x; i < 128 * 32 + 4096; i += blockDim.x) sm[i] = (float)((i * 2654435761u) >> 8);
    __syncthreads();
    uint32_t r[NCH]; uint64_t q[NCH];
    #pragma unroll
    for (int i = 0; i < NCH; i++) { r[i] = threadIdx.x * 7 + i + k0; q[i] = ((uint64_t)r[i] << 32) | (r[i] * 3u); }
    const int lane = threadIdx.x & 31;
    __syncthreads();
    long long t0 = clock64();
    #pragma unroll 1
    for (int it = 0; it < ITER; it += 4) {
        body<OP>(r, k0, k1, q, sm, lane); body<OP>(r, k0, k1, q, sm, lane);
        body<OP>(r, k0, k1, q, sm, lane); body<OP>(r, k0, k1, q, sm, lane);
    }
    long long t1 = clock64();
    __syncthreads();
    uint32_t acc = 0;
    #pragma unroll
    for (int i = 0; i < NCH; i++) acc ^= r[i] ^ (uint32_t)q[i] ^ (uint32_t)(q[i] >> 32);
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

static int g_nblk = 1;

template <int OP>
void run(const char *name, int ptx_per_body, int nthreads = 1024)
{
    uint32_t *out; long long *cyc;
    const int nblk = g_nblk;                         // one block per SM
    cudaMalloc(&out, nblk * 1024 * 4); cudaMalloc(&cyc, nblk * 8);
    size_t smem = (128 * 32 + 4096) * 4;
    cudaFuncSetAttribute(bench<OP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    bench<OP><<<nblk, nthreads, smem>>>(out, cyc, 3, 5);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0);
    bench<OP><<<nblk, nthreads, smem>>>(out, cyc, 3, 5);
    cudaEventRecord(e1);
    cudaError_t err = cudaDeviceSynchronize();
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    long long h[1024]; cudaMemcpy(h, cyc, nblk * 8, cudaMemcpyDeviceToHost);
    double avg = 0; for (int i = 0; i < nblk; i++) avg += h[i]; avg /= nblk;
    double winstr = (double)(nthreads / 32) * ITER * NCH * ptx_per_body;
    printf("%-28s thr=%4d cycles=%9.0f  warp-instr/clk/SM=%6.3f  (lane-ops/clk/SM=%7.1f)  ms=%.3f %s\n", name, nthreads, avg,
           winstr / avg, winstr * 32 / avg, ms, err == cudaSuccess ? "" : cudaGetErrorString(err));
    cudaFree(out); cudaFree(cyc);
}

int main()
{
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    printf("device %s  SMs=%d  clock=%d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
    g_nblk = p.multiProcessorCount < 1024 ? p.multiProcessorCount : 1024;
    run<0>("FADD", 1); run<1>("FMUL", 1); run<2>("FFMA", 1);
    run<6>("IADD", 1); run<7>("IMAD", 1); run<8>("LOP3", 1); run<9>("PRMT", 1); run<10>("FMNMX", 1);
    run<11>("I2F.S32", 1); run<12>("F2I.RZ", 1); run<13>("IDP4A", 1); run<14>("VABSDIFF4", 1);
    run<15>("FADD.RZ", 1); run<16>("FMUL.SAT", 1); run<17>("FSETP+SEL", 2); run<18>("SHF", 1);
    run<19>("SHL+ADD (LEA?)", 1); run<20>("I2F.U8", 1); run<21>("SUB+ADD (IADD3?)", 1); run<22>("DADD", 1);
    run<23>("SHFL.BFLY", 1);
    run<24>("mix FADD+IADD", 2); run<25>("mix FFMA+LOP3", 2); run<26>("mix FFMA+IMAD", 2); run<27>("mix FADD+PRMT", 2);
    run<30>("LDS.32 (+LOP)", 1); run<31>("LDS.128 (+3LOP)", 1); run<32>("LDS.32 LUT replicated", 1);
    run<33>("LDS.32 LUT 128-entry", 1); run<34>("LDS.64+STS.64 RMW", 2);
    run<44>("ind IDP4A | LOP3", 1); run<45>("ind IDP4A | FFMA", 1); run<46>("ind VABSDIFF4 | IDP4A", 1); run<47>("ind VABSDIFF4 | LOP3", 1);
    run<48>("ind VABSDIFF4 | FFMA", 1); run<49>("ind IADD3 | FFMA", 1); run<50>("ind IADD3 | LOP3", 1); run<51>("ind IADD3 | IDP4A", 1);
    run<52>("ind PRMT | LOP3", 1); run<53>("ind IMAD | IDP4A", 1); run<54>("ind SHF | LOP3", 1); run<55>("ind SHF | FFMA", 1);
    run<56>("ind FFMA | LOP3", 1); run<57>("ind IADD3 | IADD3", 1);
    // occupancy sensitivity of the FP pipe
    run<0>("FADD", 1, 512); run<0>("FADD", 1, 256); run<2>("FFMA", 1, 256);
    return 0;
}

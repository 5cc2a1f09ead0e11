// ptxas_vimnmx3_negate.cu -- the code-generation problem the deinterlace kernels work around (csrc/deinterlace.cu,
// DESIGN.md 4.9): Yadif's and Bwdif's spatial check, diff = max(diff, min(d-e, d-c, max(b-c, f-e)),
// -max(d-e, d-c, min(b-c, f-e))), over 2^20 random inputs, compared with the same function on the host.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false -o /tmp/vimnmx3 tools/ptxas_vimnmx3_negate.cu
//   /tmp/vimnmx3                                     (needs a GPU)
//   cuobjdump -sass /tmp/vimnmx3 | grep VIMNMX3       (no GPU needed)
//
// With CUDA 12.9 for sm_90a, variants 0 (?:) and 2 (min / max) compile the last step to one
// `VIMNMX3 Rd, mn, mx, diff, !PT` whose mx operand carries no negation: the result is max(diff, mn, +mx).  On an H100
// 80GB HBM3 both gave 344076 wrong results of 1048576, e.g. diff=74 c=236 e=41 d=205 b=186 f=171 -> 164 (right: 74).
// Variant 1 ((a + b +- |a - b|) / 2) and variant 3 (the negated maximum written as the minimum of the negated terms,
// what the kernels use) gave none.
#include <cstdio>
#include <cstdlib>
__host__ __device__ __forceinline__ int tmax(int a, int b) { return a > b ? a : b; }
__host__ __device__ __forceinline__ int tmin(int a, int b) { return a < b ? a : b; }
__host__ __device__ __forceinline__ int amax(int a, int b) { return (a + b + abs(a - b)) >> 1; }
__host__ __device__ __forceinline__ int amin(int a, int b) { return (a + b - abs(a - b)) >> 1; }
template <int V> __host__ __device__ int spat(int diff, int c, int e, int d, int b, int f)
{
    if (V == 0) {          // ternaries: what the kernel first had
        const int mx = tmax(d - e, tmax(d - c, tmin(b - c, f - e)));
        const int mn = tmin(d - e, tmin(d - c, tmax(b - c, f - e)));
        return tmax(diff, tmax(mn, -mx));
    } else if (V == 1) {   // (a + b +- |a - b|) / 2
        const int mx = amax(d - e, amax(d - c, amin(b - c, f - e)));
        const int mn = amin(d - e, amin(d - c, amax(b - c, f - e)));
        return amax(diff, amax(mn, -mx));
    } else if (V == 3) {   // min / max, the negated maximum written as the minimum of the negated terms
        const int nmx = min(e - d, min(c - d, max(c - b, e - f)));
        const int mn = min(d - e, min(d - c, max(b - c, f - e)));
        return max(diff, max(mn, nmx));
    } else {               // CUDA min / max
        const int mx = max(d - e, max(d - c, min(b - c, f - e)));
        const int mn = min(d - e, min(d - c, max(b - c, f - e)));
        return max(diff, max(mn, -mx));
    }
}
template <int V> __global__ void k(const int *in, int *out, int n)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int *p = in + 6 * i;
    out[i] = spat<V>(p[0], p[1], p[2], p[3], p[4], p[5]);
}
int main()
{
    const int n = 1 << 20;
    int *h = (int *)malloc(6 * n * sizeof(int)), *o = (int *)malloc(n * sizeof(int));
    srand(1);
    for (int i = 0; i < 6 * n; i++) h[i] = rand() % 256;
    int *din, *dout;
    cudaMalloc(&din, 6 * n * sizeof(int)); cudaMalloc(&dout, n * sizeof(int));
    cudaMemcpy(din, h, 6 * n * sizeof(int), cudaMemcpyHostToDevice);
    for (int v = 0; v < 4; v++) {
        if (v == 0) k<0><<<n / 256, 256>>>(din, dout, n);
        if (v == 1) k<1><<<n / 256, 256>>>(din, dout, n);
        if (v == 2) k<2><<<n / 256, 256>>>(din, dout, n);
        if (v == 3) k<3><<<n / 256, 256>>>(din, dout, n);
        cudaMemcpy(o, dout, n * sizeof(int), cudaMemcpyDeviceToHost);
        int bad = 0, first = -1;
        for (int i = 0; i < n; i++) {
            const int *p = h + 6 * i;
            int want = tmax(p[0], tmax(tmin(p[3]-p[2], tmin(p[3]-p[1], tmax(p[4]-p[1], p[5]-p[2]))), -tmax(p[3]-p[2], tmax(p[3]-p[1], tmin(p[4]-p[1], p[5]-p[2])))));
            if (o[i] != want) { if (first < 0) first = i; bad++; }
        }
        printf("variant %d (%s): %d of %d differ", v, v == 0 ? "?:" : v == 1 ? "abs form" : v == 2 ? "min/max" : "min/max, -max as min of negations", bad, n);
        if (first >= 0) { const int *p = h + 6 * first; printf("; e.g. diff=%d c=%d e=%d d=%d b=%d f=%d -> gpu %d", p[0], p[1], p[2], p[3], p[4], p[5], o[first]); }
        printf("\n");
    }
    return 0;
}

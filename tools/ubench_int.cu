// ubench_int.cu -- issue-rate micro-benchmark of the integer instructions the line kernels are made of
// (IMAD, IMAD.HI with 64-bit addend, SHF, LEA.HI.SX32, IADD3) on one SM sub-partition set.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_int ubench_int.cu ; run: ./ubench_int
#include <cstdio>
#include <cuda_runtime.h>

#define REP 256
template <int OP>
__global__ void k(int *out, int a0, int b0, long long *cycles)
{
    int x[8];
#pragma unroll
    for (int i = 0; i < 8; i++) x[i] = a0 + i + threadIdx.x;
    int b = b0;
    long long t0 = clock64();
#pragma unroll 1
    for (int r = 0; r < REP; r++) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            if (OP == 0) x[i] = x[i] * b + 32768;                        // IMAD
            if (OP == 1) x[i] = __mulhi(x[i], b) + x[i];                 // IMAD.HI (+ add)
            if (OP == 2) x[i] = (x[i] >> 7) ^ b;                         // SHF + LOP
            if (OP == 3) x[i] = x[i] + ((x[i] * b + 32768) >> 16);       // IMAD + LEA.HI.SX32 (one pole minus the sub)
            if (OP == 4) x[i] = x[i] + (((b - x[i]) * 42156 + 32768) >> 16); // full pole
            if (OP == 5) { long long acc = ((long long) x[i] << 32) | 0x80000000ll; // pole as one high multiply
                           x[i] = (int) ((acc + (long long) (b - x[i]) * (long long) (42156 << 15) * 2) >> 32); }
            if (OP == 6) x[i] = x[i] + b;                                // IADD
            if (OP == 7) x[i] = (int) (((long long) x[i] * b) >> 16);    // IMAD.WIDE + SHF
        }
    }
    long long t1 = clock64();
    int s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) s += x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = t1 - t0;
}

template <int OP> void run(const char *name, int warps)
{
    int *out; long long *cyc, h;
    cudaMalloc(&out, 1 << 20); cudaMalloc(&cyc, 8);
    k<OP><<<1, warps * 32>>>(out, 3, 7, cyc);
    k<OP><<<1, warps * 32>>>(out, 3, 7, cyc);
    cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    // per SM sub-partition: warps/4 warps each issue REP*8 statements
    printf("%-28s warps %2d : %.2f cycles per statement per warp-scheduler slot\n", name, warps,
           (double) h / (REP * 8.0 * (warps / 4.0)));
    cudaFree(out); cudaFree(cyc);
}

int main()
{
    for (int w : {4, 16, 32}) {
        run<0>("IMAD", w); run<1>("IMAD.HI + add", w); run<2>("SHF + LOP", w); run<3>("IMAD + LEA.HI.SX32", w);
        run<4>("pole (sub, mad, lea)", w); run<5>("pole via 64-bit high mul", w); run<6>("IADD", w);
        run<7>("IMAD.WIDE + 64-bit shift", w);
    }
    return 0;
}

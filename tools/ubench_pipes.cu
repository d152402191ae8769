// ubench_pipes.cu -- which pipe the integer instructions of the kernels use on sm_90a and at what rate: every case is a loop of
// 8 independent chains per thread, 16 warps on one SM (4 per scheduler); "A + B" cases interleave two instructions -- if the
// pair costs max(A, B) they issue to different pipes, if it costs A + B they share one.  The instruction actually generated
// is whatever cuobjdump -sass shows for the case.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_pipes ubench_pipes.cu ; run: ./ubench_pipes
#include <cstdio>
#include <cuda_runtime.h>

#define REP 512
__device__ __forceinline__ int dp2a_lo(int a, int b, int c) { int d; asm volatile("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi(int a, int b, int c) { int d; asm volatile("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp4a_su(int a, int b, int c) { int d; asm volatile("dp4a.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int imad(int a, int b, int c) { int d; asm volatile("mad.lo.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int lop(int a, int b, int c) { int d; asm volatile("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int shf(int a, int b) { int d; asm volatile("shr.s32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }
__device__ __forceinline__ int prmt(int a, int b, int c) { int d; asm volatile("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int add3(int a, int b, int c) { int d; asm volatile("{ .reg .s32 t; add.s32 t, %1, %2; add.s32 %0, t, %3; }" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int vmin_relu(int a, int b) { int d; asm volatile("min.s32.relu %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }

template <int OP>
__global__ void k(int *out, int a0, int b0, int c0, long long *cycles)
{
    int x[8], y[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { x[i] = a0 + i + threadIdx.x; y[i] = a0 * 3 + i + 5 * threadIdx.x; }
    const int b = b0, c = c0;
    long long t0 = clock64();
#pragma unroll 1
    for (int r = 0; r < REP; r++) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            if (OP == 0) x[i] = imad(x[i], b, c);
            if (OP == 1) x[i] = dp2a_lo(b, x[i], x[i]);
            if (OP == 2) x[i] = dp4a_su(b, x[i], x[i]);
            if (OP == 3) x[i] = lop(x[i], b, c);
            if (OP == 4) x[i] = shf(x[i], b);
            if (OP == 5) x[i] = prmt(x[i], b, c);
            if (OP == 6) x[i] = add3(x[i], b, c);
            if (OP == 7) x[i] = vmin_relu(x[i], b);
            if (OP == 8) { x[i] = dp2a_lo(b, x[i], x[i]); y[i] = lop(y[i], b, c); }      // IDP + LOP3
            if (OP == 9) { x[i] = dp2a_lo(b, x[i], x[i]); y[i] = imad(y[i], b, c); }     // IDP + IMAD
            if (OP == 10) { x[i] = imad(x[i], b, c); y[i] = lop(y[i], b, c); }           // IMAD + LOP3
            if (OP == 11) { x[i] = lop(x[i], b, c); y[i] = shf(y[i], b); }               // LOP3 + SHF
            if (OP == 12) { x[i] = dp2a_hi(b, x[i], dp2a_lo(c, x[i], 0)); }              // the encoder's pair
            if (OP == 13) { x[i] = imad(x[i], b, c); y[i] = add3(y[i], b, c); }          // IMAD + IADD3
            if (OP == 14) { x[i] = imad(x[i], b, c); y[i] = prmt(y[i], b, c); }          // IMAD + PRMT
            if (OP == 15) { x[i] = imad(x[i], b, c); y[i] = vmin_relu(y[i], b); }        // IMAD + VIMNMX
        }
    }
    long long t1 = clock64();
    int s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) s += x[i] + y[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = t1 - t0;
}

template <int OP> void run(const char *name, int warps)
{
    int *out; long long *cyc, h;
    cudaMalloc(&out, 1 << 20); cudaMalloc(&cyc, 8);
    k<OP><<<1, warps * 32>>>(out, 3, 7, 5, cyc);
    k<OP><<<1, warps * 32>>>(out, 3, 7, 5, cyc);
    cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    printf("%-28s warps %2d : %.2f cycles per statement per scheduler\n", name, warps, (double) h / (REP * 8.0 * (warps / 4.0)));
    cudaFree(out); cudaFree(cyc);
}

int main()
{
    for (int w : {16}) {
        run<0>("IMAD", w); run<1>("IDP.2A", w); run<2>("IDP.4A", w); run<3>("LOP3", w); run<4>("SHF", w); run<5>("PRMT", w);
        run<6>("add + add (IADD3?)", w); run<7>("VIMNMX.RELU", w); run<8>("IDP.2A + LOP3", w); run<9>("IDP.2A + IMAD", w);
        run<10>("IMAD + LOP3", w); run<11>("LOP3 + SHF", w); run<12>("IDP.2A.HI(IDP.2A.LO) chain", w); run<13>("IMAD + IADD3", w);
        run<14>("IMAD + PRMT", w); run<15>("IMAD + VIMNMX", w);
    }
    return 0;
}

// ubench_pcie.cu -- how fast can SM-issued loads / stores move rows between page-locked host memory and HBM, compared with
// the copy engines?  (crtx_frames_host moves irregularly spaced rows with copy kernels, csrc/crtx.cu k_rows_gather /
// k_rows_scatter.)   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_pcie ubench_pcie.cu ; ./ubench_pcie
#include <cstdio>
#include <cuda_runtime.h>

template <int DEPTH>
__global__ void k_copy_rows(const uint4 *__restrict__ src, uint4 *__restrict__ dst, int rows, int n16, int src_stride16, int dst_stride16)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int row = blockIdx.x * (blockDim.x >> 5) + warp; row < rows; row += gridDim.x * (blockDim.x >> 5)) {
        const uint4 *s = src + (size_t) row * src_stride16;
        uint4 *d = dst + (size_t) row * dst_stride16;
        for (int i = lane; i < n16; i += 32 * DEPTH) {
            uint4 v[DEPTH];
#pragma unroll
            for (int k = 0; k < DEPTH; k++)
                if (i + 32 * k < n16) v[k] = s[i + 32 * k];
#pragma unroll
            for (int k = 0; k < DEPTH; k++)
                if (i + 32 * k < n16) d[i + 32 * k] = v[k];
        }
    }
}

static float timed(cudaStream_t st, int reps, void (*fn)(cudaStream_t, void *), void *arg)
{
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    fn(st, arg);
    cudaStreamSynchronize(st);
    cudaEventRecord(a, st);
    for (int r = 0; r < reps; r++) fn(st, arg);
    cudaEventRecord(b, st);
    cudaStreamSynchronize(st);
    float ms; cudaEventElapsedTime(&ms, a, b);
    return ms / reps;
}

struct Job { const uint4 *src; uint4 *dst; int rows, n16, ss, ds, grid, depth; size_t bytes; };
static void run_kernel(cudaStream_t st, void *p)
{
    Job *j = (Job *) p;
    if (j->depth == 4) k_copy_rows<4><<<j->grid, 256, 0, st>>>(j->src, j->dst, j->rows, j->n16, j->ss, j->ds);
    else if (j->depth == 8) k_copy_rows<8><<<j->grid, 256, 0, st>>>(j->src, j->dst, j->rows, j->n16, j->ss, j->ds);
    else k_copy_rows<13><<<j->grid, 256, 0, st>>>(j->src, j->dst, j->rows, j->n16, j->ss, j->ds);
}
static void run_memcpy(cudaStream_t st, void *p)
{
    Job *j = (Job *) p;
    cudaMemcpyAsync(j->dst, j->src, j->bytes, cudaMemcpyDefault, st);
}

int main()
{
    const int frames = 64, rows_per = 624, row_bytes = 3328, n16 = row_bytes / 16;
    const size_t img = (size_t) rows_per * row_bytes, total = img * frames;
    uint4 *h_a, *h_b, *d_a, *d_b;
    cudaHostAlloc(&h_a, total, cudaHostAllocDefault);
    cudaHostAlloc(&h_b, total, cudaHostAllocDefault);
    cudaMalloc(&d_a, total); cudaMalloc(&d_b, total);
    cudaMemset(d_a, 1, total); memset(h_a, 2, total); memset(h_b, 3, total);
    cudaStream_t s1, s2;
    cudaStreamCreate(&s1); cudaStreamCreate(&s2);
    const int rows = frames * rows_per;
    printf("%d frames of %d rows x %d B = %.1f MB per pass\n", frames, rows_per, row_bytes, total / 1e6);
    {
        Job j = { h_a, d_a, 0, 0, 0, 0, 0, 0, total };
        float ms = timed(s1, 5, run_memcpy, &j);
        printf("copy engine   H2D whole            %7.2f GB/s\n", total / ms / 1e6);
        Job k = { d_a, h_b, 0, 0, 0, 0, 0, 0, total };
        ms = timed(s1, 5, run_memcpy, &k);
        printf("copy engine   D2H whole            %7.2f GB/s\n", total / ms / 1e6);
    }
    for (int depth : { 4, 8, 13 })
        for (int grid : { 132, 132 * 4, 132 * 8 }) {
            Job g = { h_a, d_a, rows, n16, n16, n16, grid, depth, 0 };
            float ms = timed(s1, 5, run_kernel, &g);
            Job s = { d_a, h_b, rows, n16, n16, n16, grid, depth, 0 };
            float ms2 = timed(s1, 5, run_kernel, &s);
            printf("SM copy depth %2d grid %4d   H2D (loads from host) %7.2f GB/s   D2H (stores to host) %7.2f GB/s\n", depth, grid,
                   total / ms / 1e6, total / ms2 / 1e6);
        }
    { // every third row only (what a field touches), both directions at once on two streams
        Job g = { h_a, d_a, rows / 3, n16, 3 * n16, n16, 132 * 8, 8, 0 };
        Job s = { d_b, h_b, rows / 3, n16, n16, 3 * n16, 132 * 8, 8, 0 };
        cudaEvent_t a, b, c;
        cudaEventCreate(&a); cudaEventCreate(&b); cudaEventCreate(&c);
        cudaDeviceSynchronize();
        cudaEventRecord(a, s1);
        cudaStreamWaitEvent(s2, a, 0);
        for (int r = 0; r < 10; r++) { run_kernel(s1, &g); run_kernel(s2, &s); }
        cudaEventRecord(b, s1); cudaEventRecord(c, s2);
        cudaDeviceSynchronize();
        float m1, m2; cudaEventElapsedTime(&m1, a, b); cudaEventElapsedTime(&m2, a, c);
        printf("SM copy, both directions at once, every 3rd row: H2D %7.2f GB/s, D2H %7.2f GB/s\n", total / 3.0 * 10 / m1 / 1e6, total / 3.0 * 10 / m2 / 1e6);
        Job ce1 = { h_a, d_a, 0, 0, 0, 0, 0, 0, total }, ce2 = { d_b, h_b, 0, 0, 0, 0, 0, 0, total };
        cudaEventRecord(a, s1);
        cudaStreamWaitEvent(s2, a, 0);
        for (int r = 0; r < 5; r++) { run_memcpy(s1, &ce1); run_memcpy(s2, &ce2); }
        cudaEventRecord(b, s1); cudaEventRecord(c, s2);
        cudaDeviceSynchronize();
        cudaEventElapsedTime(&m1, a, b); cudaEventElapsedTime(&m2, a, c);
        printf("copy engines, both directions at once:            H2D %7.2f GB/s, D2H %7.2f GB/s\n", total * 5 / m1 / 1e6, total * 5 / m2 / 1e6);
        // mixed: gather by SM + D2H by copy engine, and the reverse
        cudaEventRecord(a, s1);
        cudaStreamWaitEvent(s2, a, 0);
        for (int r = 0; r < 6; r++) { run_kernel(s1, &g); run_kernel(s1, &g); run_kernel(s1, &g); run_memcpy(s2, &ce2); }
        cudaEventRecord(b, s1); cudaEventRecord(c, s2);
        cudaDeviceSynchronize();
        cudaEventElapsedTime(&m1, a, b); cudaEventElapsedTime(&m2, a, c);
        printf("SM gather (every 3rd row) + copy-engine D2H:      H2D %7.2f GB/s, D2H %7.2f GB/s\n", total * 6 / m1 / 1e6, total * 6 / m2 / 1e6);
    }
    { // what crtx_frames_host could do: source rows by the SM gather (236 of 624 rows per frame), decoded rows by the copy
      // engine as five strided 2-D copies per frame (624 rows / 240 lines: the written rows repeat every 13 rows), at once
        const int pitch = row_bytes;
        cudaEvent_t a, b, c;
        cudaEventCreate(&a); cudaEventCreate(&b); cudaEventCreate(&c);
        const int starts[5] = { 0, 2, 5, 7, 10 }, widths[5] = { 1, 2, 1, 2, 2 }; // rows written per 13-row period (scanlines 1)
        for (int mode = 0; mode < 3; mode++) {
            Job g = { h_a, d_a, frames * 236, n16, 0, n16, 132 * 8, 8, 0 };
            cudaDeviceSynchronize();
            cudaEventRecord(a, s1);
            cudaStreamWaitEvent(s2, a, 0);
            const int reps = 6;
            for (int r = 0; r < reps; r++) {
                if (mode != 1) { // gather: row y of the compact image <- row (y * 624) / 236 of the frame (k_rows_gather's pattern, approximated by stride)
                    g.ss = n16 * 624 / 236; // average stride; the kernel reads rows at src + row * ss
                    run_kernel(s1, &g);
                }
                if (mode != 0)
                    for (int f = 0; f < frames; f++)
                        for (int q = 0; q < 5; q++)
                            cudaMemcpy2DAsync((char *) h_b + (size_t) f * img + (size_t) starts[q] * pitch, (size_t) 13 * pitch,
                                              (char *) d_b + (size_t) f * img + (size_t) starts[q] * pitch, (size_t) 13 * pitch,
                                              (size_t) widths[q] * pitch, 48, cudaMemcpyDeviceToHost, s2);
            }
            cudaEventRecord(b, s1); cudaEventRecord(c, s2);
            cudaDeviceSynchronize();
            float m1, m2; cudaEventElapsedTime(&m1, a, b); cudaEventElapsedTime(&m2, a, c);
            const double up = (double) frames * 236 * row_bytes * reps, down = (double) frames * 384 * row_bytes * reps;
            printf("mode %d (%s): H2D rows %7.2f GB/s (%.1f us/frame)   D2H rows by 2-D copy engine %7.2f GB/s (%.1f us/frame)\n", mode,
                   mode == 0 ? "SM gather alone" : mode == 1 ? "2-D copies alone" : "both at once", mode != 1 ? up / m1 / 1e6 : 0.0,
                   mode != 1 ? m1 * 1e3 / (frames * reps) : 0.0, mode != 0 ? down / m2 / 1e6 : 0.0, mode != 0 ? m2 * 1e3 / (frames * reps) : 0.0);
        }
    }
    { // the other pairing: source rows by the copy engine (five strided 2-D copies per frame, one row of every 13-row period
      // each: 240 of 624 rows) while the decoded rows leave by the SM scatter (384 of 624 rows per frame)
        const int pitch = row_bytes;
        cudaEvent_t a, b, c;
        cudaEventCreate(&a); cudaEventCreate(&b); cudaEventCreate(&c);
        const int starts[5] = { 0, 2, 5, 7, 10 };
        for (int mode = 0; mode < 3; mode++) {
            Job sc = { d_b, h_b, frames * 384, n16, n16, n16 * 624 / 384, 132 * 8, 8, 0 };
            cudaDeviceSynchronize();
            cudaEventRecord(a, s1);
            cudaStreamWaitEvent(s2, a, 0);
            const int reps = 6;
            for (int r = 0; r < reps; r++) {
                if (mode != 1) run_kernel(s1, &sc);
                if (mode != 0)
                    for (int f = 0; f < frames; f++)
                        for (int q = 0; q < 5; q++)
                            cudaMemcpy2DAsync((char *) d_a + (size_t) f * img + (size_t) starts[q] * pitch, (size_t) 13 * pitch,
                                              (char *) h_a + (size_t) f * img + (size_t) starts[q] * pitch, (size_t) 13 * pitch,
                                              (size_t) pitch, 48, cudaMemcpyHostToDevice, s2);
            }
            cudaEventRecord(b, s1); cudaEventRecord(c, s2);
            cudaDeviceSynchronize();
            float m1, m2; cudaEventElapsedTime(&m1, a, b); cudaEventElapsedTime(&m2, a, c);
            const double down = (double) frames * 384 * row_bytes * reps, up = (double) frames * 240 * row_bytes * reps;
            printf("pairing B mode %d (%s): D2H rows by SM scatter %7.2f GB/s (%.1f us/frame)   H2D rows by 2-D copy engine %7.2f GB/s (%.1f us/frame)\n", mode,
                   mode == 0 ? "SM scatter alone" : mode == 1 ? "2-D copies alone" : "both at once", mode != 1 ? down / m1 / 1e6 : 0.0,
                   mode != 1 ? m1 * 1e3 / (frames * reps) : 0.0, mode != 0 ? up / m2 / 1e6 : 0.0, mode != 0 ? m2 * 1e3 / (frames * reps) : 0.0);
        }
    }
    return 0;
}

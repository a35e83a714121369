// Issue rate of each FP64 mma.sync shape on the current GPU: every warp issues 8 independent accumulator chains back to
// back from registers (no memory traffic).  Prints one JSON line per shape.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/dmma_shapes scripts/dmma_shapes.cu && /tmp/dmma_shapes
#include <cstdio>
#include <cuda_runtime.h>

template <int SHAPE>  // 0: m8n8k4, 1: m16n8k4, 2: m16n8k8, 3: m16n8k16
__global__ void __launch_bounds__(256) mma_loop(double *out, int iters, double seed)
{
    double c[8][4] = {};
    double a[8], b[4];
    for (int i = 0; i < 8; ++i) a[i] = seed * (threadIdx.x + i);
    for (int i = 0; i < 4; ++i) b[i] = seed * (threadIdx.x - i);
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (SHAPE == 0)
                asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                             : "+d"(c[j][0]), "+d"(c[j][1]) : "d"(a[0]), "d"(b[0]));
            else if (SHAPE == 1)
                asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                             : "+d"(c[j][0]), "+d"(c[j][1]), "+d"(c[j][2]), "+d"(c[j][3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
            else if (SHAPE == 2)
                asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                             : "+d"(c[j][0]), "+d"(c[j][1]), "+d"(c[j][2]), "+d"(c[j][3])
                             : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
            else
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                             "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                             : "+d"(c[j][0]), "+d"(c[j][1]), "+d"(c[j][2]), "+d"(c[j][3])
                             : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                               "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
        }
    }
    double s = 0;
    for (int j = 0; j < 8; ++j) s += c[j][0] + c[j][1] + c[j][2] + c[j][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int SHAPE>
static void run(const char *name, double fma_per_mma, int sms, double *out)
{
    const int iters = 4096, blocks = sms * 2, threads = 256;
    mma_loop<SHAPE><<<blocks, threads>>>(out, 16, 1e-3);  // warm-up
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0);
    mma_loop<SHAPE><<<blocks, threads>>>(out, iters, 1e-3);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    const double flops = 2.0 * fma_per_mma * 8.0 * iters * (blocks * threads / 32.0);
    printf("{\"shape\": \"%s\", \"ms\": %.3f, \"tflops\": %.2f, \"err\": \"%s\"}\n", name, ms, flops / ms * 1e-9,
           cudaGetErrorString(cudaGetLastError()));
}

int main()
{
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    double *out = nullptr;
    cudaMalloc(&out, sizeof(double) * sms * 2 * 256);
    run<0>("m8n8k4", 8 * 8 * 4, sms, out);
    run<1>("m16n8k4", 16 * 8 * 4, sms, out);
    run<2>("m16n8k8", 16 * 8 * 8, sms, out);
    run<3>("m16n8k16", 16 * 8 * 16, sms, out);
    cudaFree(out);
    return 0;
}

// Issue-rate microbenchmark for the instruction mix of the tensor-core MLP epilogue (csrc/mppi_mlp_tc.cuh): how many
// lanes per clock per SM do MUFU.EX2 / MUFU.RCP / MUFU.TANH / F2FP (cvt.rn.bf16x2.f32) / FFMA sustain, alone and
// mixed?  Decides how the tanh of that epilogue is built (2 MUFU vs 1 MUFU + FMA-pipe work).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/ubench_pipes scripts/ubench/pipes.cu && /tmp/ubench_pipes
#include <cstdio>
#include <cuda_runtime.h>

#define ITERS 2048
#define UN 8

template <int OP> __device__ __forceinline__ void op(float& x, float& y) {
    if (OP == 0) asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(x));
    if (OP == 1) asm volatile("rcp.approx.ftz.f32 %0, %0;" : "+f"(x));
    if (OP == 2) asm volatile("tanh.approx.f32 %0, %0;" : "+f"(x));
    if (OP == 3) { unsigned r; asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(x), "f"(y)); x = __uint_as_float(r << 16); }
    if (OP == 4) asm volatile("fma.rn.f32 %0, %0, %1, %1;" : "+f"(x) : "f"(y));
    if (OP == 5) {   // tanh via ex2 + rcp (the kernel's "exact" form, slimmed): 2 MUFU + 3 FMA-pipe
        float t;
        asm volatile("mul.f32 %0, %1, 0f4038AA3B;" : "=f"(t) : "f"(x));          // 2 log2(e)
        asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(t));
        asm volatile("add.f32 %0, %0, 0f3F800000;" : "+f"(t));
        asm volatile("rcp.approx.ftz.f32 %0, %0;" : "+f"(t));
        asm volatile("fma.rn.f32 %0, %1, 0fC0000000, 0f3F800000;" : "=f"(x) : "f"(t));
    }
    if (OP == 6) {   // tanh via polynomial 2^f on the FMA pipe + MUFU.RCP: 1 MUFU + ~12 FMA/ALU
        float yv, n, f, p;
        asm volatile("mul.f32 %0, %1, 0f4038AA3B;" : "=f"(yv) : "f"(x));
        asm volatile("min.f32 %0, %0, 0f42FA0000;" : "+f"(yv));                 // 125
        asm volatile("max.f32 %0, %0, 0fC2FA0000;" : "+f"(yv));
        asm volatile("add.f32 %0, %1, 0f4B400000;" : "=f"(n) : "f"(yv));        // round to nearest via 1.5 * 2^23
        int ni = __float_as_int(n);
        asm volatile("sub.f32 %0, %0, 0f4B400000;" : "+f"(n));
        asm volatile("sub.f32 %0, %1, %2;" : "=f"(f) : "f"(yv), "f"(n));
        p = 1.535336188319500e-4f;
        p = fmaf(p, f, 1.339887440266574e-3f);
        p = fmaf(p, f, 9.618437357674640e-3f);
        p = fmaf(p, f, 5.550332471162809e-2f);
        p = fmaf(p, f, 2.402264791363012e-1f);
        p = fmaf(p, f, 6.931472028550421e-1f);
        p = fmaf(p, f, 1.0f);
        float e = __int_as_float(__float_as_int(p) + (ni << 23));
        e += 1.0f;
        asm volatile("rcp.approx.ftz.f32 %0, %0;" : "+f"(e));
        x = fmaf(e, -2.0f, 1.0f);
    }
}

template <int OP> __global__ void bench(float* out, long long* clk) {
    float v[UN], w = 1.0001f + threadIdx.x * 1e-7f;
#pragma unroll
    for (int u = 0; u < UN; ++u) v[u] = 0.1f + 0.01f * u + threadIdx.x * 1e-6f;
    __syncthreads();
    long long t0 = clock64();
    for (int i = 0; i < ITERS; ++i) {
#pragma unroll
        for (int u = 0; u < UN; ++u) op<OP>(v[u], w);
    }
    long long t1 = clock64();
    float s = 0;
#pragma unroll
    for (int u = 0; u < UN; ++u) s += v[u];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) clk[blockIdx.x] = t1 - t0;
}

template <int OP> void run(const char* name, int warps_per_sm) {
    float* out;
    long long* clk;
    int nb = 0;
    cudaDeviceGetAttribute(&nb, cudaDevAttrMultiProcessorCount, 0);     // one CTA per SM
    cudaMalloc(&out, nb * 1024 * 4);
    cudaMalloc(&clk, nb * 8);
    bench<OP><<<nb, warps_per_sm * 32>>>(out, clk);
    bench<OP><<<nb, warps_per_sm * 32>>>(out, clk);
    cudaDeviceSynchronize();
    long long h[1024];
    cudaMemcpy(h, clk, nb * 8, cudaMemcpyDeviceToHost);
    double c = 0;
    for (int i = 0; i < nb; ++i) c += (double)h[i];
    c /= nb;
    double ops = (double)ITERS * UN * warps_per_sm * 32;
    printf("%-34s warps/SM %2d: %7.1f lane-ops/clk/SM  (%6.2f clk per warp-op per SMSP)\n", name, warps_per_sm, ops / c,
           c / ((double)ITERS * UN * warps_per_sm / 4.0));
    cudaFree(out);
    cudaFree(clk);
}

int main() {
    for (int w : {4, 8, 16}) {
        run<0>("MUFU.EX2", w);
        run<1>("MUFU.RCP", w);
        run<2>("MUFU.TANH", w);
        run<3>("F2FP.BF16 (cvt.rn.bf16x2.f32)", w);
        run<4>("FFMA", w);
        run<5>("tanh = ex2 + rcp (2 MUFU + 3)", w);
        run<6>("tanh = poly 2^f + rcp (1 MUFU + ~14)", w);
    }
    return 0;
}

// chain_bench.cu — cycles per step of the birth-death recurrence for ONE warp (latency floor of a long chain).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o chain_bench chain_bench.cu
#include <cuda_runtime.h>
#include <cstdio>
struct Recip { double b, yh, yl; };
__device__ __forceinline__ double div_recip(double a, const Recip& r) {
    double t = __dmul_rn(a, r.yl);
    double q0 = __fma_rn(a, r.yh, t);
    double res = __fma_rn(-r.b, q0, a);
    return __fma_rn(res, r.yh, q0);
}
// the tail steps of the solver: S = 0 the generic division of a = RN(p*lam) (a -> t -> q0 -> r -> q), S = 1 the low
// word taken from p with the Markstein correction (a -> q0 -> r -> q), S = 2 the same without the correction, exact
// for a float32 divisor (a -> q0; wva_device.cuh step_rate)
template <int S>
__device__ __forceinline__ double step(double p, double lam, double c, const Recip& r) {
    if (S == 0) return div_recip(__dmul_rn(p, lam), r);
    const double a = __dmul_rn(p, lam);
    const double q0 = __fma_rn(a, r.yh, __dmul_rn(p, c));
    if (S == 2) return q0;
    return __fma_rn(__fma_rn(-r.b, q0, a), r.yh, q0);
}
__global__ void pass1(double lam, Recip r, int steps, double* out, long long* cyc) {
    double p = 1.0, sum = 1.0;
    long long t0 = clock64();
    for (int n = 0; n < steps; n += 4) {
#pragma unroll
        for (int u = 0; u < 4; ++u) { p = div_recip(__dmul_rn(p, lam), r); sum = __dadd_rn(sum, p); }
    }
    long long t1 = clock64();
    out[threadIdx.x] = sum + p;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void pass2(double lam, Recip r, Recip z, int steps, double* out, long long* cyc) {
    double p = 1.0, acc = 0.0, di = 1.0, pn = 0.0;
    long long t0 = clock64();
    for (int n = 0; n < steps; n += 4) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const double a_ = __dmul_rn(p, lam);
            pn = div_recip(p, z);
            p = div_recip(a_, r);
            acc = __dadd_rn(acc, __dmul_rn(di, pn));
            di = __dadd_rn(di, 1.0);
        }
    }
    long long t1 = clock64();
    out[threadIdx.x] = acc + p + pn;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void pass1_checked(double lam, Recip r, int steps, unsigned lo, unsigned span, double* out, long long* cyc) {
    double p = 1.0, sum = 1.0;
    int n = 0;
    long long t0 = clock64();
    while (n + 4 <= steps && (((unsigned)__double2hiint(p)) - lo) < span) {
#pragma unroll
        for (int u = 0; u < 4; ++u) { p = div_recip(__dmul_rn(p, lam), r); sum = __dadd_rn(sum, p); }
        n += 4;
    }
    long long t1 = clock64();
    out[threadIdx.x] = sum + p + n;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
template <int S>
__global__ void pass1_vote16(double lam, Recip r, int steps, unsigned lo, unsigned span, int nh, double* out, long long* cyc) {
    const double c = __dmul_rn(lam, r.yl);
    double p = 1.0, sum = 1.0;
    int n = 300;
    long long t0 = clock64();
    while (__all_sync(__activemask(), n > nh + 1 && n >= 24 && n + 16 <= steps && (((unsigned)__double2hiint(p)) - lo) < span)) {
#pragma unroll
        for (int u = 0; u < 16; ++u) { p = step<S>(p, lam, c, r); sum = __dadd_rn(sum, p); }
        n += 16;
    }
    long long t1 = clock64();
    out[threadIdx.x] = sum + p + n;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
template <int S>
__global__ void pass2_vote16(double lam, Recip r, Recip z, int steps, unsigned lo, unsigned span, int nh, double* out, long long* cyc) {
    const double c = __dmul_rn(lam, r.yl);
    double p = 1.0, acc = 0.0, di = 1.0, pn = 0.0;
    int i = 300;
    long long t0 = clock64();
    while (__all_sync(__activemask(), i > nh + 1 && i + 16 <= steps && (((unsigned)__double2hiint(p)) - lo) < span)) {
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            pn = div_recip(p, z);
            p = step<S>(p, lam, c, r);
            acc = __dadd_rn(acc, __dmul_rn(di, pn));
            di = __dadd_rn(di, 1.0);
        }
        i += 16;
    }
    long long t1 = clock64();
    out[threadIdx.x] = acc + p + pn + i;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

// ---- contention: W warps per SM all running the same kernel (grid = one CTA of W warps per SM) ----
__global__ void op_chain(int kind, int steps, double x, double* out) {
    double a = 1.0 + threadIdx.x * 1e-9, b = x;
    for (int n = 0; n < steps; n += 8) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            if (kind == 0) a = __fma_rn(a, b, x);
            else if (kind == 1) a = __dmul_rn(a, b);
            else a = __dadd_rn(a, b);
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a;
}
template <class F>
static double time_ms(F f) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    f(); cudaDeviceSynchronize();
    cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); return ms;
}
static void contention(double* out, long long* cyc, Recip r, Recip z, int sms, double ghz) {
    const int steps = 40000;
    const int ws[] = {1, 2, 4, 8, 12, 16, 24, 32};
    printf("warps/SM (4 per sub-partition at 16) : cycles/step pass1, pass2 for steps 0 / 1 / 2 | cycles per dependent op DFMA, DMUL, DADD\n");
    for (int w : ws) {
        double m1[3], m2[3];
        m1[0] = time_ms([&] { pass1_vote16<0><<<sms, 32 * w>>>(1.0, r, steps, 0x20000000u, 0x50000000u, 255, out, cyc); });
        m2[0] = time_ms([&] { pass2_vote16<0><<<sms, 32 * w>>>(1.0, r, z, steps, 0x20000000u, 0x50000000u, 255, out, cyc); });
        m1[1] = time_ms([&] { pass1_vote16<1><<<sms, 32 * w>>>(1.0, r, steps, 0x20000000u, 0x50000000u, 255, out, cyc); });
        m2[1] = time_ms([&] { pass2_vote16<1><<<sms, 32 * w>>>(1.0, r, z, steps, 0x20000000u, 0x50000000u, 255, out, cyc); });
        m1[2] = time_ms([&] { pass1_vote16<2><<<sms, 32 * w>>>(1.0, r, steps, 0x20000000u, 0x50000000u, 255, out, cyc); });
        m2[2] = time_ms([&] { pass2_vote16<2><<<sms, 32 * w>>>(1.0, r, z, steps, 0x20000000u, 0x50000000u, 255, out, cyc); });
        double k[3];
        for (int kind = 0; kind < 3; ++kind) k[kind] = time_ms([&] { op_chain<<<sms, 32 * w>>>(kind, steps * 8, 1.0000001, out); });
        const double cs = 1e-3 * ghz * 1e9 / (steps - 300);
        printf("%2d : %.1f %.1f / %.1f %.1f / %.1f %.1f | %.2f %.2f %.2f\n", w, m1[0] * cs, m2[0] * cs, m1[1] * cs, m2[1] * cs,
               m1[2] * cs, m2[2] * cs,
               k[0] * 1e-3 * ghz * 1e9 / (steps * 8), k[1] * 1e-3 * ghz * 1e9 / (steps * 8), k[2] * 1e-3 * ghz * 1e9 / (steps * 8));
    }
}
int main() {
    double* out; long long* cyc;
    int sms = 0, khz = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    cudaMalloc(&out, (size_t)sms * 1024 * 8); cudaMallocManaged(&cyc, 8);
    Recip r{1.0009765625, 0.0, 0.0}; r.yh = 1.0 / r.b; r.yl = (1.0 - r.b * r.yh) / r.b;
    Recip z{3.7, 0.0, 0.0}; z.yh = 1.0 / z.b; z.yl = (1.0 - z.b * z.yh) / z.b;
    const int steps = 40000;
    pass1<<<1, 32>>>(1.0, r, steps, out, cyc); cudaDeviceSynchronize();
    pass1<<<1, 32>>>(1.0, r, steps, out, cyc); cudaDeviceSynchronize();
    printf("pass 1 (recurrence + sum)            : %.1f cycles/step\n", (double)cyc[0] / steps);
    pass1_checked<<<1, 32>>>(1.0, r, steps, 0x20000000u, 0x50000000u, out, cyc); cudaDeviceSynchronize();
    printf("pass 1 + window test every 4 steps   : %.1f cycles/step\n", (double)cyc[0] / steps);
    pass2<<<1, 32>>>(1.0, r, z, steps, out, cyc); cudaDeviceSynchronize();
    printf("pass 2 (recurrence + normalise + acc): %.1f cycles/step\n", (double)cyc[0] / steps);
    for (int s = 0; s < 3; ++s) {
        const char* name[] = {"generic division", "step, corrected", "step, rate (no correction)"};
        auto p1 = s == 0 ? pass1_vote16<0> : s == 1 ? pass1_vote16<1> : pass1_vote16<2>;
        auto p2 = s == 0 ? pass2_vote16<0> : s == 1 ? pass2_vote16<1> : pass2_vote16<2>;
        p1<<<1, 32>>>(1.0, r, steps, 0x20000000u, 0x50000000u, 255, out, cyc); cudaDeviceSynchronize();
        p1<<<1, 32>>>(1.0, r, steps, 0x20000000u, 0x50000000u, 255, out, cyc); cudaDeviceSynchronize();
        printf("pass 1, vote + 16-step blocks, %-27s: %.1f cycles/step\n", name[s], (double)cyc[0] / (steps - 300));
        p2<<<1, 32>>>(1.0, r, z, steps, 0x20000000u, 0x50000000u, 255, out, cyc); cudaDeviceSynchronize();
        printf("pass 2, vote + 16-step blocks, %-27s: %.1f cycles/step\n", name[s], (double)cyc[0] / (steps - 300));
    }
    pass1_vote16<0><<<1, 1>>>(1.0, r, steps, 0x20000000u, 0x50000000u, 255, out, cyc); cudaDeviceSynchronize();
    printf("pass 1, vote + 16-step blocks, 1 lane: %.1f cycles/step\n", (double)cyc[0] / (steps - 300));
    pass1_vote16<0><<<1, 20>>>(1.0, r, steps, 0x20000000u, 0x50000000u, 255, out, cyc); cudaDeviceSynchronize();
    printf("pass 1, vote + 16-step blocks, 20 lanes: %.1f cycles/step\n", (double)cyc[0] / (steps - 300));
    pass1<<<1, 1>>>(1.0, r, steps, out, cyc); cudaDeviceSynchronize();
    printf("pass 1 (no vote), 1 lane             : %.1f cycles/step\n", (double)cyc[0] / steps);
    contention(out, cyc, r, z, sms, khz * 1e-6);
    return 0;
}

// wva_device.cuh — device-side restatement of pkg/analyzer for sm_90a.
//
// Arithmetic contract: bit-identical to the Go reference on amd64 (binary32/64, RNE, no
// FMA contraction).  Every float/double operation of the reference is issued here as an
// explicitly rounded intrinsic (__fmul_rn, __dadd_rn, ...) so the compiler can neither
// contract nor reorder it; the translation unit is also compiled with -fmad=false.
//
// The one place where the instruction sequence differs from the reference is IEEE
// division by a value that is reused many times (the state-dependent service rate and
// the normalising sum).  There the quotient is produced from a pre-computed double-word
// reciprocal, which yields the correctly rounded quotient — the same bits as the
// reference's DIVSD — in 2 dependent FP64 ops for a float32 service rate and 4 (with a
// Markstein correction) for the double sum, instead of the ~10-op generic division
// sequence (see DESIGN.md "Exact division").
#pragma once
#include <math_constants.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace wva {

// ---------------------------------------------------------------------------
// Go builtin min/max on float32 (NaN-propagating, -0 < +0).
// ---------------------------------------------------------------------------
__device__ __forceinline__ float go_minf(float a, float b) {
    if (isnan(a) || isnan(b)) return __int_as_float(0x7fc00000);
    if (a == 0.0f && b == 0.0f) return signbit(a) ? a : b;
    return a < b ? a : b;
}
__device__ __forceinline__ float go_maxf(float a, float b) {
    if (isnan(a) || isnan(b)) return __int_as_float(0x7fc00000);
    if (a == 0.0f && b == 0.0f) return signbit(a) ? b : a;
    return a > b ? a : b;
}
// Go int(float64) on amd64 (CVTTSD2SQ): "integer indefinite" on NaN / overflow.
__device__ __forceinline__ long long go_f64_to_int(double x) {
    if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return LLONG_MIN;
    return (long long)x;
}

// ---------------------------------------------------------------------------
// Service-time model: pkg/analyzer/queueanalyzer.go:257-266, 296-302, 99-118.
// ---------------------------------------------------------------------------
struct QParams {
    float alpha, beta, gamma, delta;
    int in_tok, out_tok;
};

__device__ __forceinline__ float prefill_time(const QParams& q, float batch) {  // :257-262
    if (q.in_tok == 0) return 0.0f;
    float t = __fmul_rn(q.delta, (float)q.in_tok);
    t = __fmul_rn(t, batch);
    return __fadd_rn(q.gamma, t);
}
__device__ __forceinline__ float decode_time(const QParams& q, float batch) {  // :264-266
    return __fadd_rn(q.alpha, __fmul_rn(q.beta, batch));
}
__device__ __forceinline__ float effective_concurrency(const QParams& q, float avg_serv_time, int max_batch) {
    float tokens = (float)(q.out_tok - 1);  // :296-302
    float base = __fadd_rn(q.gamma, __fmul_rn(q.alpha, tokens));
    float numerator = __fsub_rn(avg_serv_time, base);
    float denominator = __fadd_rn(__fmul_rn(q.delta, (float)q.in_tok), __fmul_rn(q.beta, tokens));
    float n = __fdiv_rn(numerator, denominator);
    return go_minf(go_maxf(n, 0.0f), (float)max_batch);
}
// servRate[n-1], n >= 1: BuildModel, queueanalyzer.go:104-113
__device__ __forceinline__ float serv_rate(const QParams& q, int n) {
    float fn = (float)n;
    float prefill = prefill_time(q, fn);
    int num_decode = q.out_tok - 1;
    if (q.in_tok == 0 && q.out_tok == 1) num_decode = 1;
    float decode = __fmul_rn((float)num_decode, decode_time(q, fn));
    return __fdiv_rn(fn, __fadd_rn(prefill, decode));
}
// RateRange (req/sec) from servRate[0] and servRate[N-1]: queueanalyzer.go:116-118
__device__ __forceinline__ float rate_min_of(float s1) { return __fmul_rn(__fmul_rn(s1, 0.001f), 1000.0f); }
__device__ __forceinline__ float rate_max_of(float sN) {
    return __fmul_rn(__fmul_rn(sN, __fsub_rn(1.0f, 0.001f)), 1000.0f);
}

// ---------------------------------------------------------------------------
// Exact division by a reused divisor.
// ---------------------------------------------------------------------------
struct Recip {  // b with its double-word reciprocal yh + yl ~= 1/b (yh = RN(1/b))
    double b, yh, yl;
};
__device__ __forceinline__ Recip make_recip(double b) {
    Recip r;
    r.b = b;
    r.yh = __ddiv_rn(1.0, b);
    double e = __fma_rn(-b, r.yh, 1.0);  // exact: yh is the correctly rounded reciprocal
    r.yl = __ddiv_rn(e, b);
    return r;
}
// RN(a / b).  q0 = RN(a*(yh+yl)) is a faithful quotient (pre-rounding relative error
// ~2^-104); Markstein's theorem then gives RN(q0 + RN(a - b*q0)*yh) = RN(a/b) exactly,
// provided no intermediate leaves the normal range — callers guarantee that with the
// exponent-window tests below.
__device__ __forceinline__ double div_recip(double a, const Recip& r) {
    double t = __dmul_rn(a, r.yl);
    double q0 = __fma_rn(a, r.yh, t);
    double res = __fma_rn(-r.b, q0, a);
    return __fma_rn(res, r.yh, q0);
}
// Division by a service rate.  The rates are float32 values (servRate is []float32 in the reference), and for a
// divisor with a 24-bit significand q0 = RN(a*yh + RN(a*yl)) is already RN(a/b): a/b - m, for any rounding midpoint
// m = O * 2^g between doubles (O odd, 54 bits), has the nonzero integer numerator of (a - b*m) / b, and b*m has a
// 78-bit odd part that a cannot match, so a/b lies at least ~2^-78 (relative) from every midpoint, while the
// FMA's exact sum a*yh + t is within ~2^-103 of a/b.  Both lie strictly between the same two midpoints, so the
// Markstein correction of div_recip can never change q0 and is dropped (proof in DESIGN.md "Exact division").
// Preconditions: the divisor is a float32 value, and the exponent windows below keep a, t and q0 normal.  The
// first is carried by the type: a RateRecip is built only from a float (make_rate_recip) or read back from a
// table that make_rate_recip filled (load_recip); a double divisor (the normalising sum) stays a Recip.
struct RateRecip {
    double b, yh, yl;
};
__device__ __forceinline__ RateRecip make_rate_recip(float rate) {
    const Recip r = make_recip((double)rate);
    RateRecip s;
    s.b = r.b;
    s.yh = r.yh;
    s.yl = r.yl;
    return s;
}
// RN(a / b) for a float32-valued b: dependent chain t -> q0 (two operations)
__device__ __forceinline__ double div_rate(double a, const RateRecip& r) {
    return __fma_rn(a, r.yh, __dmul_rn(a, r.yl));
}
// One step of the recurrence, RN(RN(p * lam) / b), with the low-word product taken from p instead of from
// a = RN(p * lam): t = RN(p * c), c = RN(lam * yl), runs in parallel with a, so the dependent chain is
// a -> q0 (two operations).  t only has to be accurate to a few ulps: its error enters the FMA's sum at
// ~2^-105 of the quotient, far inside the 2^-78 margin above.  Used where lam and the divisor are loop
// constants (the tail).
__device__ __forceinline__ double step_rate(double p, double lam, double c, const RateRecip& r) {
    return __fma_rn(__dmul_rn(p, lam), r.yh, __dmul_rn(p, c));
}

// math.Pow(x, n) for an integer n >= 0 as the Go standard library computes it (src/math/pow.go: binary powering on
// the Frexp mantissa, exponent carried in an integer, Ldexp at the end): IEEE double multiplies / adds and exact bit
// manipulation only, so a host restatement of the same algorithm gives the same bits (that is how the tests check it).
// Used by the closed-form MM1KModel only.
__device__ __forceinline__ double go_ldexp(double frac, long long e) {
    if (frac == 0.0 || isinf(frac) || isnan(frac)) return frac;
    unsigned long long x = (unsigned long long)__double_as_longlong(frac);
    long long ex = (long long)((x >> 52) & 0x7ffull);
    if (ex == 0) {
        frac = __dmul_rn(frac, 4503599627370496.0);
        x = (unsigned long long)__double_as_longlong(frac);
        ex = (long long)((x >> 52) & 0x7ffull) - 52;
    }
    e += ex - 1023;
    if (e < -1075) return copysign(0.0, frac);
    if (e > 1023) return frac < 0.0 ? -CUDART_INF : CUDART_INF;
    double m = 1.0;
    if (e < -1022) {
        e += 53;
        m = 1.0 / 9007199254740992.0;
    }
    x &= ~(0x7ffull << 52);
    x |= (unsigned long long)(e + 1023) << 52;
    return __dmul_rn(m, __longlong_as_double((long long)x));
}
__device__ __forceinline__ double go_pow_uint(double x, long long n) {
    if (n == 0 || x == 1.0) return 1.0;
    if (n == 1) return x;
    if (isnan(x)) return x;
    if (x == 0.0) return (n & 1) ? x : 0.0;
    if (isinf(x)) return (x < 0.0 && (n & 1)) ? -CUDART_INF : CUDART_INF;
    double a1 = 1.0;
    long long ae = 0;
    // Frexp: mantissa in [0.5, 1), exact
    unsigned long long xb = (unsigned long long)__double_as_longlong(x);
    long long xe = (long long)((xb >> 52) & 0x7ffull);
    if (xe == 0) {  // subnormal: normalise first
        const double xn = __dmul_rn(x, 4503599627370496.0);
        xb = (unsigned long long)__double_as_longlong(xn);
        xe = (long long)((xb >> 52) & 0x7ffull) - 52;
    }
    xe -= 1022;
    double x1 = __longlong_as_double((long long)((xb & ~(0x7ffull << 52)) | (1022ull << 52)));
    for (long long i = n; i != 0; i >>= 1) {
        if (xe < -(1 << 12) || (1 << 12) < xe) {
            ae += xe;
            break;
        }
        if (i & 1) {
            a1 = __dmul_rn(a1, x1);
            ae += xe;
        }
        x1 = __dmul_rn(x1, x1);
        xe <<= 1;
        if (x1 < 0.5) {
            x1 = __dadd_rn(x1, x1);
            xe--;
        }
    }
    return go_ldexp(a1, ae);
}

// Exponent windows (high 32 bits of the double).  With lambda and the service rates in [2^-60, 2^60], p in
// [2^-280, 2^880) keeps every intermediate of the step's reciprocal division normal (the largest is q0 < 2^1000) and
// the normalising sum below 2^900; the division by the sum additionally needs p / sum >= 2^-960 (so that the low-word
// product is either normal or negligible): pass 2 raises its lower bound to sum * 2^-960 when the sum is that large
// (derivation in DESIGN.md).  Round 1 stopped at 2^600 / 2^620: chains of N = 512 near saturation peak above 2^600
// and spent their tails outside the 16-step blocks.
#define WVA_HI(e) ((unsigned)((1023 + (e)) << 20))
__device__ __forceinline__ bool in_window(double p, unsigned lo, unsigned hi) {
    return ((unsigned)__double2hiint(p) - lo) < (hi - lo);
}
constexpr unsigned kHiPLo = WVA_HI(-280);
constexpr int kPHiExp = 880, kPHiExpNarrow = 600;
constexpr unsigned kHiPHi = WVA_HI(kPHiExp), kHiPHiNarrow = WVA_HI(kPHiExpNarrow);
constexpr unsigned kHiPnSpan = (unsigned)(960 << 20);  // pass 2: p >= 2^(E(sum) - 960)
constexpr unsigned kHiRateLo = WVA_HI(-60);
constexpr unsigned kHiRateHi = WVA_HI(60);
constexpr unsigned kHiSumLo = WVA_HI(0);
constexpr unsigned kHiSumHi = WVA_HI(900), kHiSumHiNarrow = WVA_HI(620);
constexpr unsigned kHiRowSumHi = WVA_HI(620);  // solve_row shares a chain only below this (its pass 2 keeps the fixed window)

// ---------------------------------------------------------------------------
// MM1ModelStateDependent: pkg/analyzer/mm1modelstatedependent.go:38-116.
//
// The reference stores p[0..K] and makes four passes over it.  Here nothing is stored:
// pass 1 runs the recurrence p[n+1] = (p[n]*lambda)/servRate[min(n,N-1)] keeping only
// the running sum (same summation order as :93-105); pass 2 re-runs the identical
// recurrence (identical roundings, so identical p[n]), normalises each p[n] by the sum
// (:108-112) and accumulates sum(i*p[i]) and sumP in the reference's order (:47-55).
//
// Exact early termination.  Once the chain is past its mode (lambda below every
// remaining service rate, so p is non-increasing from there on) and p[j] has dropped
// below 2^-78 * min(p[0], p[1]), every later term is a no-op in all three float64
// accumulations of the reference: sum >= p[0] = 1, sumP >= p[0]/sum, and
// sum(i*p[i]/sum) >= p[1]/sum while i < 2^23, so each remaining addend is below half an
// ulp of its accumulator; and float32(p[K]/sum) < 2^-25 makes 1 - float32(p[K]) == 1.
// Skipping those steps therefore changes no output bit (proof in DESIGN.md).  A chain
// that underflows to exactly 0 ends the same way.
//
// The overflow-rescale branches (:84-89, :96-104) cannot be reproduced without the
// stored vector; when a value leaves the safe window the solve reports kSolveBail and
// the caller re-runs the cell on the stored-vector fallback (solve_stored below).
// ---------------------------------------------------------------------------
enum { kSolveOk = 0, kSolveBail = 1 };

struct ModelStats {  // queuemodel.go:10-19 + mm1kmodel.go:15 + mm1modelstatedependent.go:12
    float throughput, avg_resp_time, avg_wait_time, avg_serv_time, avg_num_in_servers;
    float tail_rate;  // servRate[N-1] as the solver read it (solve_shared_t only; RateRange.Max follows from it)
};

// ---------------------------------------------------------------------------
// Shared-table solver (grid, size and sweep kernels), structured for issue efficiency.  The hot loops contain only the recurrence: one merged
// exponent-window test per step covers "p is negligible / zero / tiny / too large"; the
// reciprocal triple stays in registers and is re-loaded only while n <= N-1 (table entry
// N-1 is the tail, so no select between head and tail values is needed); everything rare
// (exit test, exact division for tiny p, bail-out) lives in an outer handler.
// tab: 4 doubles per entry {servRate[n], yh, yl, suffix-min}, at least N entries.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void load_recip(const double* __restrict__ tab, int n, RateRecip& r) {
    const double2 t0 = *(const double2*)(tab + 4 * n);
    r.b = t0.x;
    r.yh = t0.y;
    r.yl = tab[4 * n + 2];
}

// Table column 4 holds two float32 values: [0] min(servRate[n..]) (suffix minimum; 0 if any rate is NaN),
// [1] max(servRate[0..n]) (prefix maximum).  Both are exact (the rates are float32 values).
__device__ __forceinline__ float tab_suffix_min(const double* tab, int n) { return ((const float*)(tab + 4 * n + 3))[0]; }
__device__ __forceinline__ float tab_prefix_max(const double* tab, int n) { return ((const float*)(tab + 4 * n + 3))[1]; }
// lambda clearly below m (16 float32 ulps of margin): every later step shrinks p
__device__ __forceinline__ bool rate_below(float lambda, float m) {
    return __float_as_uint(lambda) + 16u < __float_as_uint(m) && lambda > 0.0f && m > 0.0f;
}
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

// Fast-window test on the high word: lo <= hi(p) < lo + span.
#define WVA_FASTWIN(p, lo, span) ((((unsigned)__double2hiint(p)) - (lo)) < (span))

// STAGED (grid_kernel): when the 32 lanes of a full warp read the SAME pair table (they usually do: an
// item is cut from one pair's cells) the head of both passes runs from a 32-entry window of the table
// that the warp stages in shared memory (`tbuf`, 1 KB per warp) with one coalesced load per 32 steps,
// the next window prefetched meanwhile.  Per-lane global loads two steps ahead of their use leave
// most of the L2 latency exposed (every table entry is its own 32-byte sector); the staged window takes
// the L2 trip off the dependent chain (tools/head_bench.cu compares the ways of feeding a chain).
// The FIRST window holds 64 entries (steps 1..64), loaded together with the lane's tail entry and the window
// constants in one batch at the top of the solve, so a short item (most of them: batch sizes below 64) makes ONE
// trip to L2 for everything it reads; pass 2 re-uses that window when the whole head fits in it (hmax <= 64).
// Later windows are 32 entries, prefetched in registers as before.  `tbuf` holds kStagedSlots entries.
__device__ __forceinline__ void dev_cp_async16(void* smem_dst, const void* gmem_src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}
// The float32 tail of mm1modelstatedependent.go:56-66 from avgNumInSystem (acc), avgNumInServers (in_serv) and
// p[K] / sum (pnK, 0 when the chain ended early).
__device__ __forceinline__ void stats_epilogue(double acc, double in_serv, double pnK, float lambda, ModelStats& st) {
    st.avg_num_in_servers = (float)in_serv;
    const float avg_num_in_system = (float)acc;
    st.throughput = __fmul_rn(lambda, __fsub_rn(1.0f, (float)pnK));
    st.avg_resp_time = __fdiv_rn(avg_num_in_system, st.throughput);
    st.avg_serv_time = __fdiv_rn(st.avg_num_in_servers, st.throughput);
    float w = __fsub_rn(st.avg_resp_time, st.avg_serv_time);
    if (w < 0.0f) w = 0.0f;
    st.avg_wait_time = w;
}
// True when every real y with |y - x| <= E rounds to the same float32 as x: (float)x is a normal float32 below
// FLT_MAX and [x - E, x + E] lies strictly between the two rounding midpoints next to it (exact doubles: the mean of
// two neighbouring float32 values; below a power of two the lower one is half as far away).  The ends of the
// interval are rounded outwards.
__device__ __forceinline__ bool f32_decided(double x, double E) {
    const double ax = fabs(x);
    const float f = __double2float_rn(ax);
    const unsigned fb = __float_as_uint(f);
    if (!(fb >= 0x00800000u && fb < 0x7f7fffffu)) return false;  // 0, subnormal, FLT_MAX, inf, NaN
    const double fd = (double)f;
    const double m_hi = __dmul_rn(__dadd_rn(fd, (double)__uint_as_float(fb + 1u)), 0.5);
    const double m_lo = __dmul_rn(__dadd_rn(fd, (double)__uint_as_float(fb - 1u)), 0.5);
    return __dsub_rd(ax, E) > m_lo && __dadd_ru(ax, E) < m_hi;
}
// One-pass bounds (DESIGN.md §3.2b): c·u with u = 2^-53 and c = 1 + 2^-16 absorbing the second-order terms, and an
// absolute slack for the states whose quotient p[i]/sum or i·q[i] is subnormal.
constexpr double kOnePassCu = 0x1p-53 * (1.0 + 0x1p-16);
constexpr double kOnePassAbs = 0x1p-1000;

constexpr int kStagedFirst = 64;   // entries in the first staged window
constexpr int kStagedSlots = 96;   // window slots of tbuf: pass 2 may index up to (hmax - 1) + 31 <= 94 when it re-uses the window
constexpr int kStagedTbufD = kStagedSlots * 4 + 128;  // doubles per warp: the window, then one 32-byte tail entry per lane
// WIDE: the windows of the comment above kHiPLo.  grid_kernel's instantiation (STAGED) keeps the round-1 windows
// (2^600 / 2^620, fixed pass-2 bound): its batch sizes stay below what needs more, and the extra pass-2 set-up
// perturbs its register allocation; everything else (size path, sweep, row solve callers) is WIDE.
template <int PF = 10, bool STAGED = false, bool WIDE = !STAGED>
__device__ __noinline__ int solve_shared_t(const double* __restrict__ tab, int N, int K, float lambda, ModelStats& st,
                                           double* __restrict__ tbuf = nullptr) {
    constexpr unsigned kHiPHi = WIDE ? wva::kHiPHi : kHiPHiNarrow;   // shadow the namespace constants
    constexpr unsigned kHiSumHi = WIDE ? wva::kHiSumHi : kHiSumHiNarrow;
    constexpr int kPHiExp = WIDE ? wva::kPHiExp : kPHiExpNarrow;
    constexpr bool ONEPASS = STAGED;  // pass 1 also accumulates sum(i*p[i]) and decides the float32 outputs (§3.2b)
    const unsigned warp_mask = __activemask();
    const double lam = (double)lambda;
    const int nh = N - 1;
    RateRecip A, B;  // reciprocal triples of two consecutive steps (software-pipelined table loads)
    // staged head: full warp, one table.  Everything the solve reads from the table is requested here in one
    // batch: the first 64-entry window, the lane's tail entry (T stays in registers for the whole solve) and
    // entry 0.
    bool staged = false;
    int hmax = 0, hmin = 0;
    // The tail entry servRate[N-1] is needed wherever a loop hands over to the next one.  Holding it in registers
    // for the whole solve cost the pure-tail loops six registers and ptxas a worse schedule (more cycles per
    // state); re-loading it from the table at every hand-over was one of the dependent trips
    // to L2 this version removes.  So a staged solve parks it in shared memory — one 32-byte slot per lane in the
    // window's own entry format, so that a head group in which some lanes are already past their head selects the
    // ADDRESS it reads (window slot or own tail slot) instead of selecting three doubles — and WVA_LOAD_TAIL brings
    // it back with two LDS; a solve that is not staged reads the table as before.
    double4* const tsave4 = STAGED ? reinterpret_cast<double4*>(tbuf + kStagedSlots * 4) + (threadIdx.x & 31) : nullptr;
#define WVA_LOAD_TAIL(R)                                                    \
    if (STAGED && staged) {                                                 \
        const double4 t4_ = *tsave4;                                        \
        (R).b = t4_.x;                                                      \
        (R).yh = t4_.y;                                                     \
        (R).yl = t4_.z;                                                     \
    } else {                                                                \
        load_recip(tab, nh, R);                                             \
    }
    if (STAGED) {
        staged = warp_mask == 0xffffffffu && __all_sync(0xffffffffu, tab == (const double*)__shfl_sync(0xffffffffu, (unsigned long long)tab, 0));
        if (staged) {
            hmax = __reduce_max_sync(0xffffffffu, nh);
            hmin = __reduce_min_sync(0xffffffffu, nh);
            // the first window goes straight from the table into shared memory (cp.async: holding its 64 bytes per
            // lane in registers across the prologue made ptxas allocate the pure-tail loops worse)
            const double4* tab4 = reinterpret_cast<const double4*>(tab);
            const int lane = threadIdx.x & 31;
            double4* tb0 = reinterpret_cast<double4*>(tbuf);
            const double4* s0 = tab4 + min(1 + lane, hmax);
            const double4* s1 = tab4 + min(33 + lane, hmax);
            dev_cp_async16(tb0 + lane, s0);
            dev_cp_async16(reinterpret_cast<char*>(tb0 + lane) + 16, reinterpret_cast<const char*>(s0) + 16);
            dev_cp_async16(tb0 + 32 + lane, s1);
            dev_cp_async16(reinterpret_cast<char*>(tb0 + 32 + lane) + 16, reinterpret_cast<const char*>(s1) + 16);
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
    }
    load_recip(tab, 0, A);
    load_recip(tab, nh, B);
    const double tail_b = B.b;
    st.tail_rate = (float)tail_b;
    if (STAGED && staged) {
        *tsave4 = make_double4(B.b, B.yh, B.yl, 0.0);
    }
    bool bail = !in_window(lam, kHiRateLo, kHiRateHi) || !in_window(tail_b, kHiRateLo, kHiRateHi) ||
                !in_window(A.b, kHiRateLo, kHiRateHi);
    const bool tail_mono = rate_below(lambda, (float)tail_b);

    double p = bail ? 0.0 : div_rate(lam, A);  // p[1]; RN(1*lambda) = lambda
    if (!(p >= 0.0) || (unsigned)__double2hiint(p) >= kHiPHi) bail = true;
    const double p1 = p;
    unsigned thr_hi = 0;
    if (K < (1 << 23)) thr_hi = (unsigned)__double2hiint(__dmul_rn(fmin(1.0, p1), 0x1p-78));
    // merged fast window [max(thr, 2^-280), 2^880): inside it the step is a plain reciprocal step
    const unsigned lo_eff = thr_hi > kHiPLo ? thr_hi : kHiPLo;
    const unsigned span_eff = kHiPHi - lo_eff;

    // 4-step blocks with ONE window test: a step multiplies p by lambda/servRate[.] which lies in
    // [lambda/max rate, lambda/min rate] = [2^e_lo, 2^e_hi) (exponent arithmetic, conservative), so if
    // p starts a block inside [2^-279 / 2^(3 e_lo), 2^600 / 2^(3 max(e_hi,0))) it stays inside the
    // validity window of the reciprocal division for the whole block.  A chain that becomes negligible
    // inside a block simply runs to the end of the block: those states add nothing.
    unsigned blk_lo = 1, blk_span = 0;  // empty window = blocks disabled
    unsigned blk16_lo = 1, blk16_span = 0;
    int e_lo_w = 0;  // lower exponent bound of one step's factor (pass 2 re-derives its block windows from it)
    {
        const float smax = tab_prefix_max(tab, nh), smin = tab_suffix_min(tab, 0);
        if (!bail && smin > 0.0f && smax >= smin) {
            // lambda/smax >= 2^(El - Ex - 1),  lambda/smin < 2^(El - En + 1)   (E = biased float32 exponents)
            const int El = (int)(__float_as_uint(lambda) >> 23), Ex = (int)(__float_as_uint(smax) >> 23),
                      En = (int)(__float_as_uint(smin) >> 23);
            const int e_lo = El - Ex - 1, e_hi = El - En + 1;
            e_lo_w = e_lo;
            const int lo_exp = -279 - 3 * (e_lo < 0 ? e_lo : 0), hi_exp = kPHiExp - 3 * (e_hi > 0 ? e_hi : 0);
            if (lo_exp < hi_exp && lo_exp > -1000 && hi_exp > -1000) {
                const unsigned lo4 = WVA_HI(lo_exp), hi4 = WVA_HI(hi_exp);
                blk_lo = lo4 > lo_eff ? lo4 : lo_eff;
                blk_span = hi4 > blk_lo ? hi4 - blk_lo : 0;
            }
            // the same for 16-step blocks (15 unchecked steps)
            const int lo_exp16 = -279 - 15 * (e_lo < 0 ? e_lo : 0), hi_exp16 = kPHiExp - 15 * (e_hi > 0 ? e_hi : 0);
            if (lo_exp16 < hi_exp16 && lo_exp16 > -1000 && hi_exp16 > -1000) {
                const unsigned lo16 = WVA_HI(lo_exp16), hi16 = WVA_HI(hi_exp16);
                blk16_lo = lo16 > lo_eff ? lo16 : lo_eff;
                blk16_span = hi16 > blk16_lo ? hi16 - blk16_lo : 0;
            }
        }
    }

    // ---- pass 1 -----------------------------------------------------------------
    double sum = __dadd_rn(1.0, p);
    // ONEPASS: mom = sum(i*p[i]) (one FMA per state, dw = i), with sum and mom kept at state min(N, last state) in
    // sum_N / mom_N
    double mom = p, dw = 2.0, sum_N = sum, mom_N = p;
    int j_end = K + 1;
    {
        int n = 1;  // p holds p[n]
        const int n_stop = bail ? 0 : K;
        if (STAGED && staged) {
            // steps n < nh read entry n from the window, later steps the lane's own tail entry; all lanes
            // hold the same n (they advance together or leave together).  A window in which every lane
            // is still in its head (the usual case: grid_sort_cands keeps cells of one pair and similar
            // length together) needs no per-lane select.
            const double4* tab4 = reinterpret_cast<const double4*>(tab);
            double4* tb = reinterpret_cast<double4*>(tbuf);
            const int lane = threadIdx.x & 31;
            bool ok = true;
#define WVA_SP1_GROUP(SEL)                                                                                        \
    _Pragma("unroll") for (int u = 0; u < 4; ++u) {                                                               \
        const double4 e = *((SEL) && !(n < nh) ? (const double4*)tsave4 : (const double4*)(tb + (k + u)));       \
        RateRecip R;                                                                                              \
        R.b = e.x;                                                                                                \
        R.yh = e.y;                                                                                               \
        R.yl = e.z;                                                                                               \
        p = div_rate(__dmul_rn(p, lam), R);                                                                       \
        sum = __dadd_rn(sum, p);                                                                                  \
        if constexpr (ONEPASS) {                                                                                  \
            mom = __fma_rn(dw, p, mom);                                                                           \
            dw = __dadd_rn(dw, 1.0);                                                                              \
        }                                                                                                         \
        ++n;                                                                                                      \
        if constexpr (ONEPASS) { if (n <= N) { sum_N = sum; mom_N = mom; } }                                      \
    }
#define WVA_SP1(W)                                                                                                \
    _Pragma("unroll 1") for (int k = 0; k < (W); k += 4) {                                                        \
        if (n >= hmax) break; /* every lane is past its head: the pure-tail loops below take over */             \
        if (!__all_sync(0xffffffffu, n + 4 <= n_stop && WVA_FASTWIN(p, blk_lo, blk_span))) { ok = false; break; } \
        if (n + 4 <= hmin) { WVA_SP1_GROUP(false) } else { WVA_SP1_GROUP(true) }                                  \
    }
            // first window: entries 1..64 in slots 0..63 (slot k holds the entry of step 1 + k)
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncwarp();
            double4 nxt;  // later windows travel in registers
            if (kStagedFirst + 1 < hmax) nxt = tab4[min(kStagedFirst + 1 + lane, hmax)];
            WVA_SP1(kStagedFirst)
            for (int n0 = kStagedFirst + 1; ok && n0 < hmax; n0 += 32) {
                __syncwarp();
                tb[lane] = nxt;
                __syncwarp();
                if (n0 + 32 < hmax) nxt = tab4[min(n0 + 32 + lane, hmax)];
                WVA_SP1(32)
            }
#undef WVA_SP1_GROUP
#undef WVA_SP1
        }
        // invariant at the top of the loop: A = triple of step n, B = triple of step n+1 (the tail entry is
        // already in registers: a warp that is past its heads issues no load here)
        WVA_LOAD_TAIL(A)
        B = A;
        if (n < nh) load_recip(tab, n, A);
        if (n + 1 < nh) load_recip(tab, n + 1, B);
        while (n < n_stop) {
#define WVA_P1_STEP(R)                                                      \
    p = div_rate(__dmul_rn(p, lam), R);                                     \
    if (n < nh) load_recip(tab, n + 2 < nh ? n + 2 : nh, R);                \
    sum = __dadd_rn(sum, p);                                                \
    if constexpr (ONEPASS) {                                                \
        mom = __fma_rn(dw, p, mom);                                         \
        dw = __dadd_rn(dw, 1.0);                                            \
    }                                                                       \
    ++n;                                                                    \
    if constexpr (ONEPASS) { if (n <= N) { sum_N = sum; mom_N = mom; } }
            // Block phase.  All lanes that are still in this loop take a block path together or not at all
            // (a lane on the per-step path next to lanes on a block path would serialise the warp).
            //  * pure-tail 16-step blocks: every lane is past its table head, so a step
            //    is just the recurrence and the running sum — no loads, no selects; this is where the long
            //    chains spend 10/11 of their steps;
            //  * generic 4-step blocks otherwise.
            for (;;) {
                if (__all_sync(__activemask(), n > nh + 1 && n + 16 <= n_stop && WVA_FASTWIN(p, blk16_lo, blk16_span))) {
                    const double cA = __dmul_rn(lam, A.yl);
#pragma unroll
                    for (int u = 0; u < 16; ++u) {
                        p = step_rate(p, lam, cA, A);
                        sum = __dadd_rn(sum, p);
                        if constexpr (ONEPASS) {  // n > N: past sum_N / mom_N
                            mom = __fma_rn(dw, p, mom);
                            dw = __dadd_rn(dw, 1.0);
                        }
                    }
                    n += 16;
                    continue;
                }
                if (__all_sync(__activemask(), n + 4 <= n_stop && WVA_FASTWIN(p, blk_lo, blk_span))) {
                    if (n < nh) prefetch_l1(tab + 4 * (n + PF));
                    WVA_P1_STEP(A)
                    WVA_P1_STEP(B)
                    WVA_P1_STEP(A)
                    WVA_P1_STEP(B)
                    continue;
                }
                break;
            }
            // Per-step phase: at most two checked steps, then back to the vote — the lane that failed the
            // block vote (near its end, or p about to leave the window) is usually gone by then and the
            // others must not stay on this slower path for the rest of their chain.
            if (n >= n_stop || !WVA_FASTWIN(p, lo_eff, span_eff)) goto p1_slow;
            if (n < nh) prefetch_l1(tab + 4 * (n + PF));
            WVA_P1_STEP(A)
            if (n >= n_stop || !WVA_FASTWIN(p, lo_eff, span_eff)) goto p1_slow;
            WVA_P1_STEP(B)
            continue;
#undef WVA_P1_STEP
        p1_slow:
            if (n >= n_stop) break;
            // p[n] is outside the fast window
            const unsigned hp = (unsigned)__double2hiint(p);
            if (hp < thr_hi && (n >= nh ? tail_mono : rate_below(lambda, tab_suffix_min(tab, n)))) {
                j_end = n + 1;  // negligible and past the mode: states > n contribute nothing
                break;
            }
            if (p == 0.0) { j_end = n + 1; break; }
            if (!(p > 0.0) || hp >= kHiPHi) { bail = true; break; }
            // rare: one step outside the fast loop (exact IEEE division when p is tiny)
            WVA_LOAD_TAIL(A)
            if (n < nh) load_recip(tab, n, A);
            p = hp >= kHiPLo ? div_rate(__dmul_rn(p, lam), A) : __ddiv_rn(__dmul_rn(p, lam), A.b);
            sum = __dadd_rn(sum, p);
            if constexpr (ONEPASS) {
                mom = __fma_rn(dw, p, mom);
                dw = __dadd_rn(dw, 1.0);
            }
            ++n;
            if constexpr (ONEPASS) { if (n <= N) { sum_N = sum; mom_N = mom; } }
            WVA_LOAD_TAIL(A)
            B = A;
            if (n < nh) load_recip(tab, n, A);
            if (n + 1 < nh) load_recip(tab, n + 1, B);
        }
    }
    __syncwarp(warp_mask);
    if (!in_window(sum, kHiSumLo, kHiSumHi)) bail = true;
    if (bail) { sum = 1.0; j_end = 1; }

    // ---- pass 2 -----------------------------------------------------------------
    // reciprocal of the normalising sum: zh = RN(1/sum) must be exact, zl only needs a few
    // correct bits (it enters at 2^-53), so RN(e*zh) replaces the second IEEE division
    Recip z;
    z.b = sum;
    z.yh = __ddiv_rn(1.0, sum);
    z.yl = __dmul_rn(__fma_rn(-sum, z.yh, 1.0), z.yh);
    if constexpr (ONEPASS) {
        // Pass 1's sums with zh = RN(1/sum) in place of pass 2's exact quotients: A1 ~ acc, I1 ~ in_serv, each
        // within its bound E of pass 2's value (§3.2b).  When that decides both float32 roundings on every lane (a
        // lane that bailed has nothing to decide) the warp skips pass 2; p[K]/sum is exact either way.
        const int m1 = min(N, j_end - 1);  // the last state in sumP and acc_at_N
        const double A1 = __dmul_rn(mom, z.yh), AN = __dmul_rn(mom_N, z.yh), s1 = __dmul_rn(sum_N, z.yh);
        const double d1 = __dsub_rn(1.0, s1), dN = (double)N;
        const double I1 = __dadd_rn(AN, __dmul_rn(d1, dN));
        const double E_acc = __dadd_ru(__dmul_ru(__dmul_ru(2.0 * (double)j_end, kOnePassCu), A1), kOnePassAbs);
        double t = __dmul_ru(2.0 * (double)(m1 + 1), AN);
        t = __dadd_ru(t, __dmul_ru(__dmul_ru(dN, (double)(2 * m1 + 3)), s1));
        t = __dadd_ru(t, __dmul_ru(4.0 * dN, fabs(d1)));
        t = __dadd_ru(t, 2.0 * fabs(I1));
        const double E_in = __dadd_ru(__dmul_ru(t, kOnePassCu), kOnePassAbs);
        const bool decided = bail || (f32_decided(A1, E_acc) && f32_decided(I1, E_in));
        if (__all_sync(warp_mask, decided)) {
            double pnK = 0.0;
            if (j_end == K + 1) pnK = WVA_FASTWIN(p, kHiPLo, kHiPHi - kHiPLo) ? div_recip(p, z) : __ddiv_rn(p, sum);
            stats_epilogue(A1, I1, pnK, lambda, st);
            return bail ? kSolveBail : kSolveOk;
        }
    }
    double acc = 0.0, sum_p = z.yh, pn = 0.0, di = 1.0, acc_at_N = 0.0;
    p = p1;
    // pass 2 uses the same windows unless the sum is above 2^680: then the division by the sum needs
    // p >= lo2 = 2^(E(sum) - 960), states below it take the exact IEEE path (p2_slow), and the block windows' lower
    // edges move up with it (a block's unchecked steps may shrink p by 2^e_lo each)
    const unsigned sum_hi_w = (unsigned)__double2hiint(sum);
    const unsigned lo2 = (WIDE && sum_hi_w > kHiPLo + kHiPnSpan) ? sum_hi_w - kHiPnSpan : kHiPLo;
    const unsigned span2 = kHiPHi - lo2;
    unsigned blk2_lo = blk_lo, blk2_span = blk_span, blk16b_lo = blk16_lo, blk16b_span = blk16_span;
    if (WIDE && lo2 > kHiPLo) {
        const unsigned dn = e_lo_w < 0 ? (unsigned)(-e_lo_w) : 0u;
        const unsigned lo4n = lo2 + ((3u * dn + 1u) << 20), lo16n = lo2 + ((15u * dn + 1u) << 20);
        if (lo4n > blk2_lo) {
            const unsigned hi4 = blk2_lo + blk2_span;
            blk2_lo = lo4n;
            blk2_span = hi4 > lo4n ? hi4 - lo4n : 0u;
        }
        if (lo16n > blk16b_lo) {
            const unsigned hi16 = blk16b_lo + blk16b_span;
            blk16b_lo = lo16n;
            blk16b_span = hi16 > lo16n ? hi16 - lo16n : 0u;
        }
    }
    __syncwarp(warp_mask);
    {
        int i = 1;  // p holds p[i]
        if (STAGED && staged) {
            // staged head of pass 2 (see pass 1): states i < nh take their step's entry from the window
            const double4* tab4 = reinterpret_cast<const double4*>(tab);
            double4* tb = reinterpret_cast<double4*>(tbuf);
            const int lane = threadIdx.x & 31;
            bool ok = true;
            // when the whole head fits in the first window of pass 1 (entry e in slot e - 1) it is still there
            const bool reuse = hmax <= kStagedFirst;
            const double4* tbp = tb;
#define WVA_SP2_GROUP(SEL)                                                                                        \
    _Pragma("unroll") for (int u = 0; u < 4; ++u) {                                                               \
        const double4 e = *((SEL) && !(i < nh) ? (const double4*)tsave4 : (const double4*)(tbp + (k + u)));      \
        RateRecip R;                                                                                              \
        R.b = e.x;                                                                                                \
        R.yh = e.y;                                                                                               \
        R.yl = e.z;                                                                                               \
        const double a_ = __dmul_rn(p, lam);                                                                      \
        pn = div_recip(p, z);                                                                                     \
        p = div_rate(a_, R);                                                                                      \
        acc = __dadd_rn(acc, __dmul_rn(di, pn));                                                                  \
        di = __dadd_rn(di, 1.0);                                                                                  \
        if (SEL) {                                                                                                \
            if (i <= N) {                                                                                         \
                sum_p = __dadd_rn(sum_p, pn);                                                                     \
                acc_at_N = acc;                                                                                   \
            }                                                                                                     \
        } else {                                                                                                  \
            sum_p = __dadd_rn(sum_p, pn); /* i < nh < N for every lane */                                         \
        }                                                                                                         \
        ++i;                                                                                                      \
    }                                                                                                             \
    if (!(SEL)) acc_at_N = acc;
#define WVA_SP2()                                                                                                 \
    _Pragma("unroll 1") for (int k = 0; k < 32; k += 4) {                                                         \
        if (i >= hmax) break; /* past every head: the pure-tail loops below take over */                         \
        if (!__all_sync(0xffffffffu, i + 4 <= j_end && WVA_FASTWIN(p, blk2_lo, blk2_span))) { ok = false; break; } \
        if (i + 4 <= hmin) { WVA_SP2_GROUP(false) } else { WVA_SP2_GROUP(true) }                                  \
    }
            double4 nxt;
            if (!reuse && i < hmax) nxt = tab4[min(i + lane, hmax)];
            for (int i0 = i; ok && i0 < hmax; i0 += 32) {
                if (reuse) {
                    tbp = tb + (i0 - 1);  // slots up to (hmax - 1) + 31 < kStagedSlots may be touched (values unused)
                } else {
                    __syncwarp();
                    tb[lane] = nxt;
                    __syncwarp();
                    if (i0 + 32 < hmax) nxt = tab4[min(i0 + 32 + lane, hmax)];
                }
                WVA_SP2()
            }
#undef WVA_SP2_GROUP
#undef WVA_SP2
        }
        // invariant at the top of the loop: A = triple of the step out of state i, B = of state i+1
        WVA_LOAD_TAIL(A)
        B = A;
        if (i < nh) load_recip(tab, i, A);
        if (i + 1 < nh) load_recip(tab, i + 1, B);
        while (i < j_end) {
#define WVA_P2_STEP(R)                                                      \
    {                                                                       \
        const double a_ = __dmul_rn(p, lam);                                \
        pn = div_recip(p, z);                                               \
        p = div_rate(a_, R); /* p[i+1] (unused after the last state) */     \
        if (i < nh) load_recip(tab, i + 2 < nh ? i + 2 : nh, R);            \
        acc = __dadd_rn(acc, __dmul_rn(di, pn));                            \
        di = __dadd_rn(di, 1.0);                                            \
        if (i <= N) {                                                       \
            sum_p = __dadd_rn(sum_p, pn);                                   \
            acc_at_N = acc;                                                 \
        }                                                                   \
        ++i;                                                                \
    }
            for (;;) {  // block phase, as in pass 1; pure-tail also needs i > N (sumP complete)
                if (__all_sync(__activemask(), i > nh + 1 && i > N && i + 16 <= j_end && WVA_FASTWIN(p, blk16b_lo, blk16b_span))) {
                    const double cA = __dmul_rn(lam, A.yl);
#pragma unroll
                    for (int u = 0; u < 16; ++u) {
                        pn = div_recip(p, z);
                        p = step_rate(p, lam, cA, A);
                        acc = __dadd_rn(acc, __dmul_rn(di, pn));
                        di = __dadd_rn(di, 1.0);
                    }
                    i += 16;
                    continue;
                }
                if (__all_sync(__activemask(), i + 4 <= j_end && WVA_FASTWIN(p, blk2_lo, blk2_span))) {
                    if (i < nh) prefetch_l1(tab + 4 * (i + PF));
                    WVA_P2_STEP(A)
                    WVA_P2_STEP(B)
                    WVA_P2_STEP(A)
                    WVA_P2_STEP(B)
                    continue;
                }
                break;
            }
            // per-step phase (see pass 1)
            if (i >= j_end || !WVA_FASTWIN(p, lo2, span2)) goto p2_slow;
            if (i < nh) prefetch_l1(tab + 4 * (i + PF));
            WVA_P2_STEP(A)
            if (i >= j_end || !WVA_FASTWIN(p, lo2, span2)) goto p2_slow;
            WVA_P2_STEP(B)
            continue;
#undef WVA_P2_STEP
        p2_slow:
            if (i >= j_end) break;
            if (p == 0.0) { pn = 0.0; break; }
            // rare: tiny p, exact IEEE divisions
            WVA_LOAD_TAIL(A)
            if (i < nh) load_recip(tab, i, A);
            pn = __ddiv_rn(p, sum);
            acc = __dadd_rn(acc, __dmul_rn(di, pn));
            di = __dadd_rn(di, 1.0);
            if (i <= N) {
                sum_p = __dadd_rn(sum_p, pn);
                acc_at_N = acc;
            }
            p = __ddiv_rn(__dmul_rn(p, lam), A.b);
            ++i;
            WVA_LOAD_TAIL(A)
            B = A;
            if (i < nh) load_recip(tab, i, A);
            if (i + 1 < nh) load_recip(tab, i + 1, B);
        }
    }
    __syncwarp(warp_mask);
    // acc_at_N tracked acc while i <= N: it holds acc at state min(N, last state)
    const double in_serv = __dadd_rn(acc_at_N, __dmul_rn(__dsub_rn(1.0, sum_p), (double)N));
    const double pnK = (j_end == K + 1) ? pn : 0.0;
    stats_epilogue(acc, in_serv, pnK, lambda, st);
#undef WVA_LOAD_TAIL
    return bail ? kSolveBail : kSolveOk;
}

// ---------------------------------------------------------------------------
// Row solve (grid): the chain of a (server, accelerator, replica level) triple with an
// "infinitely large" batch, i.e. running on the head of the table only.  If that chain ends
// (early termination or underflow to 0) at state j_last, then for EVERY batch size b >= j_last + 2
// the cell's own chain is this very chain: it reads the same rates servRate[0..j_last-1], takes the
// same head-type exit test at the same state, never reaches its tail, and every state it
// accumulates lies below N = b.  Those cells therefore share pass 1 and pass 2 outright (same
// operations in the same order, hence the same bits) and differ only in the N-dependent float
// tail, which grid_shared evaluates per cell.  Anything off the plain fast path (tiny p that
// needs IEEE division, a chain that reaches the table end, window violations) just reports
// "no sharing" and the cells go through grid_kernel as usual.
// ---------------------------------------------------------------------------
// Inlined into its two call sites so that the shared-memory call compiles to LDS (grid_order stages the
// pair's table).  Both passes run 4 steps per window test where the exponent bounds allow it
// (solve_shared_t's argument); lanes are independent rows, so there is no warp vote here.
__device__ __forceinline__ bool solve_row(const double* __restrict__ tab, int len, float lambda, double& acc_out,
                                          double& sump_out, int& j_last) {
    const double lam = (double)lambda;
    const int nh = len - 1;
    RateRecip A, B;
    load_recip(tab, 0, A);
    if (!in_window(lam, kHiRateLo, kHiRateHi) || !in_window(A.b, kHiRateLo, kHiRateHi) || nh < 2) return false;
    double p = div_rate(lam, A);
    if (!(p >= 0.0) || (unsigned)__double2hiint(p) >= kHiPHi) return false;
    const double p1 = p;
    const unsigned thr_hi = (unsigned)__double2hiint(__dmul_rn(fmin(1.0, p1), 0x1p-78));
    const unsigned lo_eff = thr_hi > kHiPLo ? thr_hi : kHiPLo;
    const unsigned span_eff = kHiPHi - lo_eff;
    // 4-step window: p may move by 2^(3 e_lo) .. 2^(3 e_hi) inside a block
    unsigned blk_lo = 1, blk_span = 0;
    {
        const float smax = tab_prefix_max(tab, nh), smin = tab_suffix_min(tab, 0);
        if (smin > 0.0f && smax >= smin) {
            const int El = (int)(__float_as_uint(lambda) >> 23), Ex = (int)(__float_as_uint(smax) >> 23),
                      En = (int)(__float_as_uint(smin) >> 23);
            const int e_lo = El - Ex - 1, e_hi = El - En + 1;
            const int lo_exp = -279 - 3 * (e_lo < 0 ? e_lo : 0), hi_exp = kPHiExp - 3 * (e_hi > 0 ? e_hi : 0);
            if (lo_exp < hi_exp && lo_exp > -1000 && hi_exp > -1000) {
                const unsigned lo4 = WVA_HI(lo_exp), hi4 = WVA_HI(hi_exp);
                blk_lo = lo4 > lo_eff ? lo4 : lo_eff;
                blk_span = hi4 > blk_lo ? hi4 - blk_lo : 0;
            }
        }
    }
    double sum = __dadd_rn(1.0, p);
    int n = 1;
    load_recip(tab, 1, A);  // triple of step n, loaded one step ahead of its use
    // a chain that becomes negligible inside a block runs to the end of the block: those states add nothing,
    // and the exit test below then sees an even smaller p at a later state of the same (decreasing) stretch
    while (n + 4 < nh && WVA_FASTWIN(p, blk_lo, blk_span)) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            load_recip(tab, n + 1, B);
            p = div_rate(__dmul_rn(p, lam), A);
            sum = __dadd_rn(sum, p);
            A = B;
            ++n;
        }
    }
    while (n < nh && WVA_FASTWIN(p, lo_eff, span_eff)) {
        load_recip(tab, n + 1 < nh ? n + 1 : nh, B);
        p = div_rate(__dmul_rn(p, lam), A);
        sum = __dadd_rn(sum, p);
        A = B;
        ++n;
    }
    if (n >= nh) return false;  // still alive at the end of the table
    const unsigned hp = (unsigned)__double2hiint(p);
    const bool negligible = hp < thr_hi && rate_below(lambda, tab_suffix_min(tab, n));
    if (!negligible && !(p == 0.0)) return false;
    if (!in_window(sum, kHiSumLo, kHiRowSumHi)) return false;  // above: no sharing, the cells take the full solver
    j_last = n;
    Recip z;
    z.b = sum;
    z.yh = __ddiv_rn(1.0, sum);
    z.yl = __dmul_rn(__fma_rn(-sum, z.yh, 1.0), z.yh);
    double acc = 0.0, sum_p = z.yh, di = 1.0;
    p = p1;
    load_recip(tab, 1, A);
    int i = 1;
    // the block window's lower edge is >= 2^-279 / 2^(3 e_lo): all four states divide inside the window
    while (i + 3 <= j_last && WVA_FASTWIN(p, blk_lo, blk_span)) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            load_recip(tab, i + 1 < nh ? i + 1 : nh, B);
            const double pn = div_recip(p, z);
            acc = __dadd_rn(acc, __dmul_rn(di, pn));
            di = __dadd_rn(di, 1.0);
            sum_p = __dadd_rn(sum_p, pn);
            p = div_rate(__dmul_rn(p, lam), A);
            A = B;
            ++i;
        }
    }
    for (; i <= j_last; ++i) {
        if (!WVA_FASTWIN(p, kHiPLo, kHiPHi - kHiPLo)) {
            if (p == 0.0) break;  // adds nothing (the cell's pass 2 stops here as well)
            return false;
        }
        load_recip(tab, i + 1 < nh ? i + 1 : nh, B);
        const double pn = div_recip(p, z);
        acc = __dadd_rn(acc, __dmul_rn(di, pn));
        di = __dadd_rn(di, 1.0);
        sum_p = __dadd_rn(sum_p, pn);
        p = div_rate(__dmul_rn(p, lam), A);
        A = B;
    }
    acc_out = acc;
    sump_out = sum_p;
    return true;
}
// Model statistics of a cell that shares its row's chain: mm1modelstatedependent.go:50-66 with
// avgNumInSystem = acc, sumP complete at i == N, p[K] negligible.
__device__ __forceinline__ void stats_from_row(double acc, double sum_p, int N, float lambda, ModelStats& st) {
    const double in_serv = __dadd_rn(acc, __dmul_rn(__dsub_rn(1.0, sum_p), (double)N));
    st.avg_num_in_servers = (float)in_serv;
    const float avg_num_in_system = (float)acc;
    st.throughput = __fmul_rn(lambda, __fsub_rn(1.0f, 0.0f));
    st.avg_resp_time = __fdiv_rn(avg_num_in_system, st.throughput);
    st.avg_serv_time = __fdiv_rn(st.avg_num_in_servers, st.throughput);
    float w = __fsub_rn(st.avg_resp_time, st.avg_serv_time);
    if (w < 0.0f) w = 0.0f;
    st.avg_wait_time = w;
}

__device__ __forceinline__ int solve_shared(const double* __restrict__ tab, int N, int K, float lambda, ModelStats& st) {
    return solve_shared_t<>(tab, N, K, lambda, st);
}
// Per-lane private tables (size path): every lane streams its own table, so prefetch much further ahead.
__device__ __forceinline__ int solve_private(const double* __restrict__ tab, int N, int K, float lambda, ModelStats& st) {
    return solve_shared_t<48>(tab, N, K, lambda, st);
}

// Stored-vector fallback: a literal restatement of computeProbabilities /
// computeStatistics on a scratch p[0..K] in global memory, including the overflow
// rescale loops.  Used only for cells the streaming solve bailed out of.  tab is the
// entry's service-rate table; column 0 is float32 servRate widened to double.
// Returns 0 ok, 2 = the reference's rescale loop would not terminate (unsupported input).
__device__ __noinline__ int solve_stored(double* p, const double* tab, int N, int K, float lambda, ModelStats& st) {
    const double lam = (double)lambda;
    p[0] = 1.0;
    const double scale = __ddiv_rn(1.7976931348623157e308, (double)K);
    for (int n = 0; n < K; ++n) {
        const double s_rate = tab[4 * (n < N ? n : N - 1)];
        double v = __ddiv_rn(__dmul_rn(p[n], lam), s_rate);
        int guard = 0;
        while (v < 0.0 || isinf(v) || isnan(v)) {
            if (++guard > 64) return 2;
            for (int i = 0; i <= n; ++i) p[i] = __ddiv_rn(p[i], scale);
            v = __ddiv_rn(__dmul_rn(p[n], lam), s_rate);
        }
        p[n + 1] = v;
    }
    double sum = 0.0;
    for (int n = 0; n <= K; ++n) {
        sum = __dadd_rn(sum, p[n]);
        if (sum < 0.0 || isinf(sum)) {
            sum = 0.0;
            for (int i = 0; i <= K; ++i) {
                p[i] = __ddiv_rn(p[i], scale);
                if (i <= n) sum = __dadd_rn(sum, p[i]);
            }
        }
    }
    for (int n = 0; n <= K; ++n) p[n] = __ddiv_rn(p[n], sum);
    double acc = 0.0, in_serv = 0.0, sum_p = p[0];
    for (int i = 1; i <= K; ++i) {
        acc = __dadd_rn(acc, __dmul_rn((double)i, p[i]));
        sum_p = __dadd_rn(sum_p, p[i]);
        if (i == N) in_serv = __dadd_rn(acc, __dmul_rn(__dsub_rn(1.0, sum_p), (double)N));
    }
    st.avg_num_in_servers = (float)in_serv;
    const float avg_num_in_system = (float)acc;
    st.throughput = __fmul_rn(lambda, __fsub_rn(1.0f, (float)p[K]));
    st.avg_resp_time = __fdiv_rn(avg_num_in_system, st.throughput);
    st.avg_serv_time = __fdiv_rn(st.avg_num_in_servers, st.throughput);
    float w = __fsub_rn(st.avg_resp_time, st.avg_serv_time);
    if (w < 0.0f) w = 0.0f;
    st.avg_wait_time = w;
    return 0;
}

// The two solves behind one signature, true when the solve succeeded: a streaming kernel solves with SharedSolve,
// and its stored-vector re-run with StoredSolve on its scratch slot, which keeps the code of the last solve.
struct SharedSolve {
    __device__ __forceinline__ bool operator()(const double* tab, int N, int K, float lambda, ModelStats& st) const {
        return solve_shared(tab, N, K, lambda, st) == kSolveOk;
    }
};
struct StoredSolve {
    double* p;
    int rc;  // solve_stored's code of the last solve
    __device__ __forceinline__ bool operator()(const double* tab, int N, int K, float lambda, ModelStats& st) {
        rc = solve_stored(p, tab, N, K, lambda, st);
        return rc == 0;
    }
};

// The entries a streaming kernel bailed on, for the stored-vector re-run.  Each path packs its entry into 64 bits
// (fb_pack for two ints).  An append past cap is counted but not stored; fb_rerun reports it.
struct FbList {
    int* count;
    unsigned long long* item;
    int cap;
};
__device__ __forceinline__ void fb_push(const FbList& l, unsigned long long item) {
    const int k = atomicAdd(l.count, 1);
    if (k < l.cap) l.item[k] = item;
}
__device__ __forceinline__ unsigned long long fb_pack(int hi, int lo) {
    return (unsigned long long)(unsigned)hi << 32 | (unsigned)lo;
}

// What a re-run kernel needs besides its path's arguments: the list, one scratch slot of Kmax + 1 doubles per
// thread (p[0..K] of solve_stored) and the two status words the host checks after the call.
struct FbRun {
    FbList list;
    double* scratch;
    int Kmax;
    int* status;    // solve_stored's code of a solve that failed
    int* overflow;  // 1: the list had more entries than its cap
};

// The re-run loop: thread `slot` takes list entries slot, slot + n_slots, ...; body(item, p) re-runs one entry on
// scratch p and returns solve_stored's code (0: ok).
template <class Body>
__device__ __forceinline__ void fb_rerun(const FbRun& r, Body&& body) {
    const int n_slots = gridDim.x * blockDim.x;
    const int slot = blockIdx.x * blockDim.x + threadIdx.x;
    int n = *r.list.count;
    if (n > r.list.cap) {
        if (slot == 0) *r.overflow = 1;
        n = r.list.cap;
    }
    double* p = r.scratch + (size_t)slot * ((size_t)r.Kmax + 1);
    for (int k = slot; k < n; k += n_slots) {
        const int rc = body(r.list.item[k], p);
        if (rc != 0) atomicExch(r.status, rc);
    }
}

// ---------------------------------------------------------------------------
// QueueAnalyzer.Analyze metrics from solved model stats: queueanalyzer.go:152-172.
// ---------------------------------------------------------------------------
struct Metrics {
    float throughput, avg_wait_time, avg_prefill_time, avg_token_time, rho, ttft;
};
__device__ __forceinline__ Metrics metrics_from(const QParams& q, int N, const ModelStats& st) {
    Metrics m;

    const float eff = effective_concurrency(q, st.avg_serv_time, N);
    m.avg_prefill_time = prefill_time(q, eff);
    m.avg_token_time = decode_time(q, eff);
    float rho = __fdiv_rn(st.avg_num_in_servers, (float)N);
    m.rho = go_minf(go_maxf(rho, 0.0f), 1.0f);
    m.throughput = __fmul_rn(st.throughput, 1000.0f);
    m.avg_wait_time = st.avg_wait_time;
    m.ttft = __fadd_rn(st.avg_wait_time, m.avg_prefill_time);
    return m;
}

// WithinTolerance: pkg/analyzer/utils.go:12-20
__device__ __forceinline__ bool within_tolerance(float x, float value, float tol) {
    if (x == value) return true;
    if (value == 0.0f || tol < 0.0f) return false;
    return fabs((double)__fdiv_rn(__fsub_rn(x, value), value)) <= (double)tol;
}

// TransitionPenalty: pkg/core/allocation.go:291-300
__device__ __forceinline__ float transition_penalty(float factor, int cur_acc, int cur_replicas, float cur_cost,
                                                    int new_acc, int new_replicas, float new_cost) {
    if (cur_acc == new_acc && cur_acc != -2) {
        if (cur_replicas == new_replicas) return 0.0f;
        return __fsub_rn(new_cost, cur_cost);
    }
    return __fadd_rn(__fmul_rn(factor, __fadd_rn(cur_cost, new_cost)), __fsub_rn(new_cost, cur_cost));
}

// The first bit pattern in (l, h] at which pred holds, given that it fails at l, holds at h and never fails again
// once it holds: a bisection over float32 bit patterns, which are ordered like the values of one sign.
template <class Pred>
__device__ __forceinline__ unsigned bits_first(unsigned l, unsigned h, Pred&& pred) {
    while (h - l > 1u) {
        const unsigned m = l + (h - l) / 2u;
        if (pred(m)) h = m;
        else l = m;
    }
    return h;
}

}  // namespace wva

/*
 * wva_oracle.c — CPU restatement of the WVA optimizer hot path (TEST INFRASTRUCTURE;
 * see wva_oracle.h for the rules about who may call this).
 *
 * Every function cites the reference file:line it follows (paths relative to the
 * reference checkout).  The restatement is deliberately literal: same operation
 * order, same float32/float64 mix, same loops (including the four passes over p[]),
 * so that its run time is an honest stand-in for the reference's CPU path and its
 * results are what Go/amd64 produces.
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -fPIC -shared (oracle/Makefile).
 */
#include "wva_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------ */
/* Go builtin semantics                                                      */
/* ------------------------------------------------------------------------ */

/* Go builtin min/max on floats: NaN if any operand is NaN; -0 < +0. */
static float go_minf(float a, float b) {
    if (isnan(a) || isnan(b)) return NAN;
    if (a == 0.0f && b == 0.0f) return signbit(a) ? a : b;
    return a < b ? a : b;
}
static float go_maxf(float a, float b) {
    if (isnan(a) || isnan(b)) return NAN;
    if (a == 0.0f && b == 0.0f) return signbit(a) ? b : a;
    return a > b ? a : b;
}
/* Go int(float64) on amd64: CVTTSD2SQ, "integer indefinite" on NaN / overflow. */
static int64_t go_f64_to_int(double x) {
    if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return INT64_MIN;
    return (int64_t)x;
}
static int64_t i64max(int64_t a, int64_t b) { return a > b ? a : b; }

static int64_t g_solves, g_states;
int64_t wvao_last_solves(void) { return g_solves; }
int64_t wvao_last_states(void) { return g_states; }

/* Queue models the oracle refused since the last call of this function (see queue_states). */
static int64_t g_unsupported;
int64_t wvao_take_unsupported(void) {
    int64_t n = g_unsupported;
    g_unsupported = 0;
    return n;
}

/* BuildModel's K = MaxBatchSize + MaxQueueSize with MaxQueueSize = N * MaxQueueToBatchRatio, in Go's 64-bit int
 * (allocation.go:88-93, queueanalyzer.go:115).  A model of 2^31 states or more has no int32 K (the analyzer here,
 * the CUDA library and the ABI all count states in int32) and would need a p[] of 16 GiB or more: it is counted
 * in g_unsupported and -1 is returned, and the caller builds nothing. */
static int queue_states(int64_t N, int ratio, int *max_queue) {
    if (N >= ((int64_t)1 << 31) || N * (1 + (int64_t)ratio) >= ((int64_t)1 << 31)) {
        g_unsupported++;
        return -1;
    }
    *max_queue = ratio < 0 ? -1 : (int)(N * ratio); /* negative: Configuration.check refuses it */
    return 0;
}

/* ------------------------------------------------------------------------ */
/* pkg/analyzer/queueanalyzer.go: service-time model                        */
/* ------------------------------------------------------------------------ */

/* queueanalyzer.go:257-262 */
float wvao_prefill_time(float gamma, float delta, int in_tokens, float batch) {
    if (in_tokens == 0) return 0;
    float t = delta * (float)in_tokens;
    t = t * batch;
    return gamma + t;
}

/* queueanalyzer.go:264-266 */
float wvao_decode_time(float alpha, float beta, float batch) {
    float t = beta * batch;
    return alpha + t;
}

/* queueanalyzer.go:296-302 */
float wvao_effective_concurrency(float avg_serv_time, float alpha, float beta, float gamma,
                                 float delta, int in_tokens, int out_tokens, int max_batch) {
    float tokens = (float)(out_tokens - 1);
    float at = alpha * tokens;
    float base = gamma + at;
    float numerator = avg_serv_time - base;
    float d1 = delta * (float)in_tokens;
    float d2 = beta * tokens;
    float denominator = d1 + d2;
    float n = numerator / denominator;
    return go_minf(go_maxf(n, 0), (float)max_batch);
}

/* ------------------------------------------------------------------------ */
/* pkg/analyzer/utils.go                                                    */
/* ------------------------------------------------------------------------ */

static const float kEpsilonSearch = 1e-6f; /* utils.go:8 */
static const int kMaxIterations = 100;     /* utils.go:9 */

/* utils.go:12-20 */
int wvao_within_tolerance(float x, float value, float tol) {
    if (x == value) return 1;
    if (value == 0 || tol < 0) return 0;
    float d = x - value;
    float q = d / value;
    return fabs((double)q) <= (double)tol;
}

/* utils.go:26-70 */
int wvao_binary_search(float xmin, float xmax, float ytarget, wvao_eval_fn eval, void *ctx,
                       float *xstar_out, int *ind_out) {
    *xstar_out = 0;
    *ind_out = 0;
    if (xmin > xmax) return 1;

    float ybounds[2];
    float xs[2] = {xmin, xmax};
    for (int i = 0; i < 2; i++) {
        if (eval(ctx, xs[i], &ybounds[i]) != 0) return 2;
        if (wvao_within_tolerance(ybounds[i], ytarget, kEpsilonSearch)) {
            *xstar_out = xs[i];
            *ind_out = 0;
            return 0;
        }
    }

    int increasing = ybounds[0] < ybounds[1];
    if ((increasing && ytarget < ybounds[0]) || (!increasing && ytarget > ybounds[0])) {
        *xstar_out = xmin;
        *ind_out = -1;
        return 0;
    }
    if ((increasing && ytarget > ybounds[1]) || (!increasing && ytarget < ybounds[1])) {
        *xstar_out = xmax;
        *ind_out = +1;
        return 0;
    }

    float xstar = 0, ystar = 0;
    for (int it = 0; it < kMaxIterations; it++) {
        float s = xmin + xmax;
        xstar = 0.5f * s;
        if (eval(ctx, xstar, &ystar) != 0) return 2;
        if (wvao_within_tolerance(ystar, ytarget, kEpsilonSearch)) break;
        if ((increasing && ytarget < ystar) || (!increasing && ytarget > ystar)) {
            xmax = xstar;
        } else {
            xmin = xstar;
        }
    }
    *xstar_out = xstar;
    *ind_out = 0;
    return 0;
}

/* ------------------------------------------------------------------------ */
/* pkg/analyzer/mm1kmodel.go — closed-form M/M/1/K (not on the production   */
/* path; restated for the reference's model tests)                          */
/* ------------------------------------------------------------------------ */

/* math.Pow for a non-negative integer exponent, restated from the Go standard library's pure-Go implementation
 * (src/math/pow.go, the only one amd64 has): special cases, then binary powering on the Frexp mantissa with the
 * exponent carried in an integer, then Ldexp.  Every operation is an IEEE double multiply/add or exact bit
 * manipulation, so the CUDA restatement (wva_device.cuh: go_pow_uint) produces the same bits.  The Go toolchain is
 * absent here: this follows the published algorithm and is NOT pinned against the Go binary; the test suite checks it
 * against libm's pow to a few ulp (tests/test_mm1k.py). */
static double go_ldexp(double frac, int64_t e) { /* src/math/ldexp.go */
    if (frac == 0 || isinf(frac) || isnan(frac)) return frac;
    uint64_t x;
    memcpy(&x, &frac, 8);
    int64_t ex = (int64_t)((x >> 52) & 0x7ff);
    if (ex == 0) { /* normalize a subnormal */
        frac *= 4503599627370496.0; /* 2^52 */
        memcpy(&x, &frac, 8);
        ex = (int64_t)((x >> 52) & 0x7ff) - 52;
    }
    e += ex - 1023;
    if (e < -1075) return copysign(0.0, frac);
    if (e > 1023) return frac < 0 ? -INFINITY : INFINITY;
    double m = 1.0;
    if (e < -1022) { /* denormal result: one rounding, in the final multiply */
        e += 53;
        m = 1.0 / 9007199254740992.0; /* 2^-53 */
    }
    x &= ~((uint64_t)0x7ff << 52);
    x |= (uint64_t)(e + 1023) << 52;
    double r;
    memcpy(&r, &x, 8);
    return m * r;
}
double wvao_go_pow_uint(double x, int64_t n) { /* math.Pow(x, float64(n)), n >= 0 */
    if (n == 0 || x == 1) return 1;
    if (n == 1) return x;
    if (isnan(x)) return x;
    if (x == 0) return (n & 1) ? x : 0.0; /* y > 0: +-0 for odd y, +0 otherwise */
    if (isinf(x)) return (x < 0 && (n & 1)) ? -INFINITY : INFINITY;
    double a1 = 1.0;
    int64_t ae = 0;
    int xe_i;
    double x1 = frexp(x, &xe_i); /* exact; frac in [0.5, 1) */
    int64_t xe = xe_i;
    for (int64_t i = n; i != 0; i >>= 1) {
        if (xe < -(1 << 12) || (1 << 12) < xe) { /* catastrophic over/underflow: Ldexp settles it */
            ae += xe;
            break;
        }
        if (i & 1) {
            a1 *= x1;
            ae += xe;
        }
        x1 *= x1;
        xe <<= 1;
        if (x1 < .5) {
            x1 += x1;
            xe--;
        }
    }
    return go_ldexp(a1, ae);
}

struct wvao_mm1k {
    int K;
    double *p;
    double sum_p;
    wvao_model_stats st;
};

wvao_mm1k *wvao_mm1k_new(int K) { /* mm1kmodel.go:19-30 */
    if (K < 0) return NULL;
    wvao_mm1k *m = (wvao_mm1k *)calloc(1, sizeof(*m));
    if (!m) return NULL;
    m->K = K;
    m->p = (double *)calloc((size_t)K + 1, sizeof(double));
    return m;
}
void wvao_mm1k_free(wvao_mm1k *m) {
    if (!m) return;
    free(m->p);
    free(m);
}
const double *wvao_mm1k_probs(const wvao_mm1k *m) { return m->p; }

/* queuemodel.go:27-37 with MM1KModel.ComputeRho (mm1kmodel.go:38-44), GetRhoMax
 * (:46-48), computeProbabilities (:51-72), computeStatistics (:75-92). */
void wvao_mm1k_solve(wvao_mm1k *m, float lambda, float mu, wvao_model_stats *out) {
    wvao_model_stats *s = &m->st;
    s->lambda = lambda;
    s->mu = mu;
    s->rho = (lambda == mu) ? 1.0f : lambda / mu;
    if ((s->rho < 0) || (s->rho >= (float)m->K) || (lambda < 0) || (mu <= 0)) {
        s->is_valid = 0;
    } else {
        s->is_valid = 1;
        for (int i = 0; i <= m->K; i++) m->p[i] = 0;
        m->sum_p = 1;
        if (s->rho == 1) {
            m->p[0] = 1 / (double)(m->K + 1);
        } else {
            m->p[0] = (1 - (double)s->rho) / (1 - wvao_go_pow_uint((double)s->rho, (int64_t)m->K + 1));
        }
        m->sum_p = 0;
        double p0 = m->p[0];
        for (int i = 0; i <= m->K; i++) {
            m->p[i] = p0 * wvao_go_pow_uint((double)s->rho, (int64_t)i);
            m->sum_p += m->p[i];
        }
        double temp = 0;
        for (int i = 0; i <= m->K; i++) {
            double t = (double)i * m->p[i];
            temp += t;
        }
        s->avg_num_in_system = (float)temp;
        s->throughput = lambda * (1 - (float)m->p[m->K]);
        s->avg_resp_time = s->avg_num_in_system / s->throughput;
        s->avg_serv_time = 1 / mu;
        s->avg_wait_time = s->avg_resp_time - s->avg_serv_time;
        if (s->avg_wait_time < 0) s->avg_wait_time = 0;
        s->avg_queue_length = s->throughput * s->avg_wait_time;
        s->sum_p = m->sum_p;
    }
    if (out) *out = *s;
}

/* ------------------------------------------------------------------------ */
/* pkg/analyzer/mm1modelstatedependent.go + queueanalyzer.go                */
/* ------------------------------------------------------------------------ */

struct wvao_analyzer {
    /* QueueAnalyzer (queueanalyzer.go:14-21) */
    int max_batch, max_queue;
    float alpha, beta, gamma, delta;
    int in_tokens, out_tokens;
    float rate_min, rate_max;
    /* MM1ModelStateDependent (mm1modelstatedependent.go:9-13) */
    int K;
    float *serv_rate; /* [max_batch] */
    double *p;        /* [K+1], zero-initialised by make() */
    wvao_model_stats st;
    int64_t solves;
    int rescale_stuck; /* set when the reference's rescale loop would not terminate */
};

/* mm1modelstatedependent.go:70-116 */
static void sd_compute_probabilities(wvao_analyzer *m) {
    double *p = m->p;
    const int K = m->K;
    const int num = m->max_batch;
    const double lam = (double)m->st.lambda;
    p[0] = 1;
    double scale = DBL_MAX / (double)K;
    double s_rate = 0;
    for (int n = 0; n < K; n++) {
        if (n < num)
            s_rate = (double)m->serv_rate[n];
        else
            s_rate = (double)m->serv_rate[num - 1];
        double t = p[n] * lam;
        p[n + 1] = t / s_rate;
        int guard = 0;
        while (p[n + 1] < 0 || isinf(p[n + 1]) || isnan(p[n + 1])) {
            /* The reference loops forever when the value never recovers (e.g. a NaN
             * input); a bounded oracle flags that instead of hanging. */
            if (++guard > 64) {
                m->rescale_stuck = 1;
                break;
            }
            for (int i = 0; i <= n; i++) p[i] /= scale;
            t = p[n] * lam;
            p[n + 1] = t / s_rate;
        }
    }
    double sum = 0;
    for (int n = 0; n <= K; n++) {
        sum += p[n];
        if (sum < 0 || isinf(sum)) {
            sum = 0;
            for (int i = 0; i <= K; i++) {
                p[i] /= scale;
                if (i <= n) sum += p[i];
            }
        }
    }
    double sum_p = 0;
    for (int n = 0; n <= K; n++) {
        p[n] /= sum;
        sum_p += p[n];
    }
    m->st.sum_p = sum_p;
    m->st.rho = 1 - (float)p[0]; /* ComputeRho :33-35 */
}

/* mm1modelstatedependent.go:38-67 */
static void sd_compute_statistics(wvao_analyzer *m) {
    sd_compute_probabilities(m);
    const double *p = m->p;
    const int K = m->K;
    const int num = m->max_batch;
    double avg_num_in_servers = 0;
    double avg_num_in_system = 0;
    double sum_p = p[0];
    for (int i = 1; i <= K; i++) {
        double t = (double)i * p[i];
        avg_num_in_system += t;
        sum_p += p[i];
        if (i == num) {
            double u = 1 - sum_p;
            u = u * (double)num;
            avg_num_in_servers = avg_num_in_system + u;
        }
    }
    wvao_model_stats *s = &m->st;
    s->avg_num_in_servers = (float)avg_num_in_servers;
    s->avg_num_in_system = (float)avg_num_in_system;
    s->throughput = s->lambda * (1 - (float)p[K]);
    s->avg_resp_time = s->avg_num_in_system / s->throughput;
    s->avg_serv_time = s->avg_num_in_servers / s->throughput;
    s->avg_wait_time = s->avg_resp_time - s->avg_serv_time;
    if (s->avg_wait_time < 0) s->avg_wait_time = 0;
    s->avg_queue_length = s->throughput * s->avg_wait_time;
}

/* QueueModel.Solve: queuemodel.go:27-37; ComputeRho reads the p[0] left by the
 * previous solve (mm1modelstatedependent.go:33-35). */
void wvao_model_solve(wvao_analyzer *m, float lambda, float mu, wvao_model_stats *out) {
    wvao_model_stats *s = &m->st;
    m->solves++;
    g_solves++;
    s->lambda = lambda;
    s->mu = mu;
    s->rho = 1 - (float)m->p[0];
    if ((s->rho < 0) || (s->rho >= (float)m->K) || (lambda < 0) || (mu <= 0)) {
        s->is_valid = 0;
    } else {
        s->is_valid = 1;
        g_states += m->K;
        sd_compute_statistics(m);
    }
    if (out) *out = *s;
}

/* NewQueueAnalyzer + BuildModel: queueanalyzer.go:87-131, checks :305-319 */
wvao_analyzer *wvao_analyzer_new(int max_batch, int max_queue, float alpha, float beta, float gamma,
                                 float delta, int in_tokens, int out_tokens) {
    if (max_batch <= 0 || max_queue < 0) return NULL; /* Configuration.check */
    if (in_tokens < 0 || out_tokens < 1) return NULL; /* RequestSize.check   */
    wvao_analyzer *qa = (wvao_analyzer *)calloc(1, sizeof(*qa));
    if (!qa) return NULL;
    qa->max_batch = max_batch;
    qa->max_queue = max_queue;
    qa->alpha = alpha;
    qa->beta = beta;
    qa->gamma = gamma;
    qa->delta = delta;
    qa->in_tokens = in_tokens;
    qa->out_tokens = out_tokens;
    qa->serv_rate = (float *)malloc(sizeof(float) * (size_t)max_batch);
    for (int n = 1; n <= max_batch; n++) {
        float prefill = wvao_prefill_time(gamma, delta, in_tokens, (float)n);
        int num_decode = out_tokens - 1;
        if (in_tokens == 0 && out_tokens == 1) num_decode = 1;
        float decode = (float)num_decode * wvao_decode_time(alpha, beta, (float)n);
        float tot = prefill + decode;
        qa->serv_rate[n - 1] = (float)n / tot;
    }
    const float eps = 0.001f; /* Epsilon :8 */
    float lambda_min = qa->serv_rate[0] * eps;
    float lambda_max = qa->serv_rate[max_batch - 1] * (1 - eps);
    qa->rate_min = lambda_min * 1000;
    qa->rate_max = lambda_max * 1000;
    qa->K = max_queue + max_batch;
    qa->p = (double *)calloc((size_t)qa->K + 1, sizeof(double));
    return qa;
}

/* NewMM1ModelStateDependent(K, servRate) (mm1modelstatedependent.go:16-24) on its own: the reference's
 * queuemodel_test.go builds models from arbitrary rate vectors, with K larger than the vector (the last rate
 * then serves every deeper state, :80-84).  Only wvao_model_solve / probs / K are meaningful on the result. */
wvao_analyzer *wvao_model_new_rates(int K, const float *serv_rate, int n) {
    if (K < 0 || n <= 0 || !serv_rate) return NULL;
    wvao_analyzer *qa = (wvao_analyzer *)calloc(1, sizeof(*qa));
    if (!qa) return NULL;
    qa->max_batch = n;
    qa->max_queue = K - n;
    qa->out_tokens = 1;
    qa->serv_rate = (float *)malloc(sizeof(float) * (size_t)n);
    for (int i = 0; i < n; i++) qa->serv_rate[i] = serv_rate[i];
    qa->K = K;
    qa->p = (double *)calloc((size_t)K + 1, sizeof(double));
    return qa;
}

void wvao_analyzer_free(wvao_analyzer *qa) {
    if (!qa) return;
    free(qa->serv_rate);
    free(qa->p);
    free(qa);
}
void wvao_analyzer_rate_range(const wvao_analyzer *qa, float *rmin, float *rmax) {
    *rmin = qa->rate_min;
    *rmax = qa->rate_max;
}
const float *wvao_analyzer_serv_rate(const wvao_analyzer *qa) { return qa->serv_rate; }
const double *wvao_analyzer_probs(const wvao_analyzer *qa) { return qa->p; }
int wvao_analyzer_K(const wvao_analyzer *qa) { return qa->K; }
int64_t wvao_analyzer_solves(const wvao_analyzer *qa) { return qa->solves; }

/* queueanalyzer.go:134-174 */
int wvao_analyze(wvao_analyzer *qa, float request_rate, wvao_metrics *out) {
    if (request_rate <= 0) return 1;
    if (request_rate > qa->rate_max) return 2;
    wvao_model_solve(qa, request_rate / 1000, 1, NULL);
    if (!qa->st.is_valid) return 3;
    float avg_num_in_serv = qa->st.avg_num_in_servers;
    float eff = wvao_effective_concurrency(qa->st.avg_serv_time, qa->alpha, qa->beta, qa->gamma,
                                           qa->delta, qa->in_tokens, qa->out_tokens, qa->max_batch);
    float prefill = wvao_prefill_time(qa->gamma, qa->delta, qa->in_tokens, eff);
    float token = wvao_decode_time(qa->alpha, qa->beta, eff);
    float rho = avg_num_in_serv / (float)qa->max_batch;
    rho = go_minf(go_maxf(rho, 0), 1);
    out->throughput = qa->st.throughput * 1000;
    out->avg_resp_time = qa->st.avg_resp_time;
    out->avg_wait_time = qa->st.avg_wait_time;
    out->avg_num_in_serv = avg_num_in_serv;
    out->avg_prefill_time = prefill;
    out->avg_token_time = token;
    out->max_rate = qa->rate_max;
    out->rho = rho;
    return 0;
}

/* queueanalyzer.go:270-279 */
int wvao_eval_ttft(wvao_analyzer *qa, float x, float *y) {
    wvao_model_solve(qa, x, 1, NULL);
    if (!qa->st.is_valid) return 1;
    float wait = qa->st.avg_wait_time;
    float eff = wvao_effective_concurrency(qa->st.avg_serv_time, qa->alpha, qa->beta, qa->gamma,
                                           qa->delta, qa->in_tokens, qa->out_tokens, qa->max_batch);
    *y = wait + wvao_prefill_time(qa->gamma, qa->delta, qa->in_tokens, eff);
    return 0;
}
/* queueanalyzer.go:283-290 */
int wvao_eval_itl(wvao_analyzer *qa, float x, float *y) {
    wvao_model_solve(qa, x, 1, NULL);
    if (!qa->st.is_valid) return 1;
    float eff = wvao_effective_concurrency(qa->st.avg_serv_time, qa->alpha, qa->beta, qa->gamma,
                                           qa->delta, qa->in_tokens, qa->out_tokens, qa->max_batch);
    *y = wvao_decode_time(qa->alpha, qa->beta, eff);
    return 0;
}
static int eval_ttft_cb(void *ctx, float x, float *y) { return wvao_eval_ttft((wvao_analyzer *)ctx, x, y); }
static int eval_itl_cb(void *ctx, float x, float *y) { return wvao_eval_itl((wvao_analyzer *)ctx, x, y); }

/* queueanalyzer.go:185-255 */
int wvao_size(wvao_analyzer *qa, const wvao_target_perf *target, wvao_target_rate *rates,
              wvao_metrics *metrics, wvao_target_perf *achieved) {
    if (target->itl < 0 || target->ttft < 0 || target->tps < 0) return 1; /* :322-329 */
    float lambda_min = qa->rate_min / 1000;
    float lambda_max = qa->rate_max / 1000;
    int ind = 0, err;

    float lambda_star_ttft = lambda_max;
    if (target->ttft > 0) {
        err = wvao_binary_search(lambda_min, lambda_max, target->ttft, eval_ttft_cb, qa,
                                 &lambda_star_ttft, &ind);
        if (ind < 0 || err != 0) return 2;
    }
    float lambda_star_itl = lambda_max;
    if (target->itl > 0) {
        err = wvao_binary_search(lambda_min, lambda_max, target->itl, eval_itl_cb, qa,
                                 &lambda_star_itl, &ind);
        if (ind < 0 || err != 0) return 3;
    }
    float lambda_star_tps = lambda_max;
    if (target->tps > 0) {
        const float ssf = 0.1f; /* StabilitySafetyFraction :11 */
        lambda_star_tps = lambda_max * (1 - ssf);
    }
    float lambda = go_minf(go_minf(lambda_star_ttft, lambda_star_itl), lambda_star_tps);
    float request_rate = lambda * 1000;
    wvao_metrics m;
    if (wvao_analyze(qa, request_rate, &m) != 0) return 4;
    if (metrics) *metrics = m;
    if (rates) {
        rates->rate_ttft = lambda_star_ttft * 1000;
        rates->rate_itl = lambda_star_itl * 1000;
        rates->rate_tps = lambda_star_tps * 1000;
    }
    if (achieved) {
        achieved->ttft = m.avg_wait_time + m.avg_prefill_time;
        achieved->itl = m.avg_token_time;
        achieved->tps = m.throughput * (float)qa->out_tokens;
    }
    return 0;
}

/* ------------------------------------------------------------------------ */
/* pkg/core                                                                 */
/* ------------------------------------------------------------------------ */

static int num_instances(const wva_fleet *f, int m, int a) { /* model.go:50-57 */
    int c = f->perf_acc_count[m * f->n_acc + a];
    return c <= 0 ? 1 : c;
}

/* allocation.go:291-300. Accelerator names compare equal iff both are the same
 * known id or both are "" (WVA_ACC_NONE); WVA_ACC_UNKNOWN never equals anything a
 * candidate can carry. */
float wvao_transition_penalty(float factor, int cur_acc, int cur_replicas, float cur_cost,
                              int new_acc, int new_replicas, float new_cost) {
    if (cur_acc == new_acc && cur_acc != WVA_ACC_UNKNOWN) {
        if (cur_replicas == new_replicas) return 0;
        return new_cost - cur_cost;
    }
    float s = cur_cost + new_cost;
    float p = factor * s;
    float d = new_cost - cur_cost;
    return p + d;
}

static void alloc_nil(wvao_alloc *o) {
    memset(o, 0, sizeof(*o));
    o->acc = WVA_ACC_NONE;
}

/* allocation.go:259-288 */
static void zero_load_allocation(const wva_fleet *f, int s, int m, int a, wvao_alloc *o) {
    const int A = f->n_acc;
    int64_t num_replicas = f->srv_min_replicas[s];
    if (num_replicas == 0) {
        alloc_nil(o);
        o->feasible = 1; /* accelerator "", everything 0 */
        return;
    }
    int max_batch = f->perf_max_batch[m * A + a];
    if (f->srv_max_batch[s] > 0) max_batch = f->srv_max_batch[s];
    int64_t total = (int64_t)num_instances(f, m, a) * num_replicas;
    float cost = f->acc_cost[a] * (float)total;
    float alpha = f->perf_alpha[m * A + a], beta = f->perf_beta[m * A + a];
    float gamma = f->perf_gamma[m * A + a], delta = f->perf_delta[m * A + a];
    float decode_time = alpha + beta;
    float bt = beta * (float)max_batch;
    float max_decode_time = alpha + bt;
    float prefill_time = gamma + delta;
    float max_serv_time = prefill_time + max_decode_time;
    float max_rate = (float)max_batch / max_serv_time;
    o->feasible = 1;
    o->acc = a;
    o->replicas = (int32_t)num_replicas;
    o->batch = max_batch;
    o->cost = cost;
    o->value = cost;
    o->itl = decode_time;
    o->ttft = prefill_time;
    o->rho = 0;
    o->max_rate = max_rate;
}

/* allocation.go:27-163 */
void wvao_create_allocation(const wva_fleet *f, int s, int a, wvao_alloc *o) {
    const int A = f->n_acc;
    alloc_nil(o);
    if (a < 0 || a >= A) return;              /* GetAccelerator == nil :42 */
    if (s < 0 || s >= f->n_servers) return;   /* GetServer == nil :47 */
    if (f->srv_arrival_rpm[s] < 0 || f->srv_in_tokens[s] < 0 || f->srv_out_tokens[s] < 0)
        return;                                /* :50-53 */
    int m = f->srv_model[s];
    if (m < 0 || m >= f->n_models) return;     /* GetModel == nil :57 */
    if (!f->perf_present[m * A + a]) return;   /* PerfData == nil :60 */
    if (!f->srv_has_target[s]) return;         /* service class / target :65-70 */

    if (f->srv_arrival_rpm[s] == 0 || f->srv_out_tokens[s] == 0) { /* :73-75 */
        zero_load_allocation(f, s, m, a, o);
        return;
    }
    int K = f->srv_out_tokens[s];
    int64_t N64;
    if (f->srv_max_batch[s] > 0) {
        N64 = f->srv_max_batch[s];
    } else {
        int64_t t = (int64_t)f->perf_max_batch[m * A + a] * (int64_t)f->perf_at_tokens[m * A + a] / K;
        N64 = t > 1 ? t : 1;
    }
    int max_queue;
    if (queue_states(N64, f->tun.max_queue_to_batch_ratio, &max_queue) != 0) return;
    int N = (int)N64;

    wvao_analyzer *qa = wvao_analyzer_new(N, max_queue, f->perf_alpha[m * A + a], f->perf_beta[m * A + a],
                                          f->perf_gamma[m * A + a], f->perf_delta[m * A + a],
                                          f->srv_in_tokens[s], K);
    if (!qa) return; /* :110-114 */

    wvao_target_perf target = {f->srv_slo_ttft[s], f->srv_slo_itl[s], f->srv_slo_tps[s]};
    wvao_metrics metrics;
    if (wvao_size(qa, &target, NULL, &metrics, NULL) != 0) { /* :126-130 */
        wvao_analyzer_free(qa);
        return;
    }
    float rate_star = metrics.throughput;

    float total_rate; /* :134-139 */
    if (target.tps == 0) {
        total_rate = f->srv_arrival_rpm[s] / 60;
    } else {
        total_rate = target.tps / (float)K;
    }
    int64_t num_replicas = go_f64_to_int(ceil((double)total_rate / (double)rate_star));
    num_replicas = i64max(num_replicas, (int64_t)f->srv_min_replicas[s]);

    int64_t total_instances = (int64_t)num_instances(f, m, a) * num_replicas; /* :144-145 */
    float cost = f->acc_cost[a] * (float)total_instances;

    float rate = total_rate / (float)num_replicas; /* :148-153 */
    if (wvao_analyze(qa, rate, &metrics) != 0) {
        wvao_analyzer_free(qa);
        return;
    }
    o->feasible = 1;
    o->acc = a;
    o->replicas = (int32_t)num_replicas;
    o->batch = N;
    o->cost = cost;
    o->value = cost;
    o->itl = metrics.avg_token_time;
    o->ttft = metrics.avg_wait_time + metrics.avg_prefill_time;
    o->rho = metrics.rho;
    o->max_rate = rate_star / 1000;
    wvao_analyzer_free(qa);
}

/* Is accelerator a a candidate for server s? server.go:70-82 */
static int is_candidate_acc(const wva_fleet *f, int s, int a) {
    if (f->srv_keep_acc[s] && f->srv_cur_acc[s] != WVA_ACC_NONE) return f->srv_cur_acc[s] == a;
    return 1;
}

/* server.go:55-67 for every server */
void wvao_calculate(const wva_fleet *f, wvao_alloc *out) {
    const int A = f->n_acc;
    g_solves = 0;
    g_states = 0;
    for (int s = 0; s < f->n_servers; s++) {
        for (int a = 0; a < A; a++) {
            wvao_alloc *o = &out[(size_t)s * A + a];
            alloc_nil(o);
            if (!is_candidate_acc(f, s, a)) continue;
            wvao_create_allocation(f, s, a, o);
            if (o->feasible) {
                /* curAllocation is never nil (server.go:49) */
                o->value = wvao_transition_penalty(f->tun.accel_penalty_factor, f->srv_cur_acc[s],
                                                   f->srv_cur_replicas[s], f->srv_cur_cost[s], o->acc,
                                                   o->replicas, o->cost);
            }
        }
    }
}

/* ------------------------------------------------------------------------ */
/* pkg/solver                                                               */
/* ------------------------------------------------------------------------ */

/* solver.go:63-79 (strict <, start at MaxFloat32; lowest acc id wins ties) */
void wvao_solve_unlimited(const wva_fleet *f, const wvao_alloc *cand, wvao_alloc *winners) {
    const int A = f->n_acc;
    for (int s = 0; s < f->n_servers; s++) {
        float min_val = FLT_MAX;
        const wvao_alloc *best = NULL;
        for (int a = 0; a < A; a++) {
            const wvao_alloc *c = &cand[(size_t)s * A + a];
            if (!c->feasible) continue;
            if (c->value < min_val) {
                min_val = c->value;
                best = c;
            }
        }
        if (best)
            winners[s] = *best;
        else
            alloc_nil(&winners[s]);
    }
}

/* cmp.Compare for float32: NaN sorts before everything, NaN == NaN */
static int cmp_f32(float a, float b) {
    int an = isnan(a), bn = isnan(b);
    if (an && bn) return 0;
    if (an) return -1;
    if (bn) return 1;
    return a < b ? -1 : (a > b ? 1 : 0);
}
static int cmp_int(int a, int b) { return a < b ? -1 : (a > b ? 1 : 0); }

typedef struct greedy_entry { /* greedy.go:16-22 */
    int server;
    int priority;
    int cur_index;
    int n_allocs;
    int *allocs; /* candidate accelerator ids, sorted by value */
    float delta;
} greedy_entry;

typedef struct greedy_ctx {
    const wva_fleet *f;
    wvao_alloc *cand;
    wvao_alloc *winners;
    int *available; /* [T] */
} greedy_ctx;

static wvao_alloc *entry_alloc(greedy_ctx *c, const greedy_entry *e, int idx) {
    return &c->cand[(size_t)e->server * c->f->n_acc + e->allocs[idx]];
}

/* greedy.go:76-85 */
static int order_func(greedy_ctx *c, const greedy_entry *a, const greedy_entry *b) {
    if (a->priority == b->priority) {
        if (a->delta == b->delta) {
            return cmp_f32(entry_alloc(c, b, b->cur_index)->value, entry_alloc(c, a, a->cur_index)->value);
        }
        return cmp_f32(b->delta, a->delta);
    }
    return cmp_int(a->priority, b->priority);
}

/* stable insertion sort (the reference's pdqsort is unstable; ties are resolved by
 * original order here = server id / accelerator id) */
static void sort_entries(greedy_ctx *c, greedy_entry **v, int n) {
    for (int i = 1; i < n; i++) {
        greedy_entry *x = v[i];
        int j = i - 1;
        while (j >= 0 && order_func(c, v[j], x) > 0) {
            v[j + 1] = v[j];
            j--;
        }
        v[j + 1] = x;
    }
}

static int units_per_replica(const wva_fleet *f, int s, int a) {
    return num_instances(f, f->srv_model[s], a) * f->acc_multiplicity[a];
}

/* greedy.go:107-166 */
static int greedy_allocate(greedy_ctx *c, greedy_entry **entries, int n, greedy_entry **unalloc) {
    int n_un = 0;
    /* entries is used as a queue [head, head+len) inside a buffer of capacity n */
    int head = 0, len = n;
    while (len > 0) {
        greedy_entry *top = entries[head];
        head++;
        len--;
        if (top->n_allocs == 0) continue;
        int s = top->server;
        wvao_alloc *alloc = entry_alloc(c, top, top->cur_index);
        int g = alloc->acc;
        if (g < 0 || g >= c->f->n_acc) continue; /* GetAccelerator == nil (acc "") */
        int t = c->f->acc_type[g];
        int count = alloc->replicas * units_per_replica(c->f, s, g);
        if (c->available[t] >= count) {
            c->available[t] -= count;
            c->winners[s] = *alloc;
        } else {
            top->cur_index++;
            if (top->cur_index + 1 < top->n_allocs) {
                top->delta = entry_alloc(c, top, top->cur_index + 1)->value -
                             entry_alloc(c, top, top->cur_index)->value;
            } else if (top->cur_index == top->n_allocs) {
                unalloc[n_un++] = top;
                continue;
            } else {
                top->delta = FLT_MAX;
            }
            /* slices.BinarySearchFunc: leftmost i with cmp(entries[i], top) >= 0 */
            int lo = 0, hi = len;
            while (lo < hi) {
                int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
                if (order_func(c, entries[head + mid], top) < 0)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            /* insert at head+lo: shift the prefix [head, head+lo) one slot left */
            head--;
            for (int k = 0; k < lo; k++) entries[head + k] = entries[head + k + 1];
            entries[head + lo] = top;
            len++;
        }
    }
    return n_un;
}

/* greedy.go:194-223 */
static void allocate_maximally(greedy_ctx *c, greedy_entry **es, int n) {
    const wva_fleet *f = c->f;
    for (int k = 0; k < n; k++) {
        greedy_entry *e = es[k];
        for (int i = 0; i < e->n_allocs; i++) {
            wvao_alloc *alloc = entry_alloc(c, e, i);
            int g = alloc->acc;
            if (g < 0 || g >= f->n_acc) continue;
            int upr = units_per_replica(f, e->server, g);
            if (upr > 0) {
                int t = f->acc_type[g];
                int max_replicas = c->available[t] / upr;
                if (alloc->replicas < max_replicas) max_replicas = alloc->replicas;
                if (max_replicas > 0) {
                    int cur = alloc->replicas;
                    float factor = (float)max_replicas / (float)cur;
                    alloc->cost = alloc->cost * factor;
                    alloc->value = alloc->value * factor;
                    alloc->replicas = max_replicas;
                    c->winners[e->server] = *alloc;
                    c->available[t] -= max_replicas * upr;
                    break;
                }
            }
        }
    }
}

/* greedy.go:239-316 */
static void allocate_equally(greedy_ctx *c, greedy_entry **es, int n) {
    const wva_fleet *f = c->f;
    typedef struct ticket {
        int present, active, acc_type, upr, num_replicas, allocated;
        wvao_alloc *final_alloc;
    } ticket;
    ticket *tk = (ticket *)calloc((size_t)n > 0 ? (size_t)n : 1, sizeof(ticket));
    int n_tickets = 0;
    for (int k = 0; k < n; k++) {
        tk[k].present = 1;
        n_tickets++;
    }
    while (n_tickets > 0) {
        for (int k = 0; k < n; k++) {
            ticket *t = &tk[k];
            greedy_entry *e = es[k];
            if (!t->present) continue;
            if (!t->active) {
                for (int i = 0; i < e->n_allocs; i++) {
                    wvao_alloc *alloc = entry_alloc(c, e, i);
                    int g = alloc->acc;
                    if (g < 0 || g >= f->n_acc) continue;
                    int upr = units_per_replica(f, e->server, g);
                    if (upr > 0 && c->available[f->acc_type[g]] >= upr) {
                        t->active = 1;
                        t->acc_type = f->acc_type[g];
                        t->upr = upr;
                        t->final_alloc = alloc;
                        break;
                    }
                }
                if (!t->active) {
                    t->present = 0;
                    n_tickets--;
                    continue;
                }
            }
            int replicas_available = c->available[t->acc_type] / t->upr;
            int allocatable = replicas_available < t->final_alloc->replicas ? replicas_available
                                                                            : t->final_alloc->replicas;
            if (allocatable > 0) {
                t->num_replicas++;
                c->available[t->acc_type] -= t->upr;
                t->allocated = 1;
            } else {
                t->present = 0;
                n_tickets--;
            }
        }
    }
    for (int k = 0; k < n; k++) {
        ticket *t = &tk[k];
        if (!t->allocated) continue;
        wvao_alloc *alloc = t->final_alloc;
        int cur = alloc->replicas;
        float factor = (float)t->num_replicas / (float)cur;
        alloc->cost = alloc->cost * factor;
        alloc->value = alloc->value * factor;
        alloc->replicas = t->num_replicas;
        c->winners[es[k]->server] = *alloc;
    }
    free(tk);
}

/* greedy.go:169-190 */
static void best_effort(greedy_ctx *c, greedy_entry **un, int n) {
    switch (c->f->saturation_policy) {
    case WVA_SAT_PRIORITY_EXHAUSTIVE:
        allocate_maximally(c, un, n);
        break;
    case WVA_SAT_PRIORITY_ROUND_ROBIN: {
        int i = 0;
        while (i < n) { /* makePriorityGroups :321-341 */
            int j = i + 1;
            while (j < n && un[j]->priority == un[i]->priority) j++;
            allocate_equally(c, un + i, j - i);
            i = j;
        }
        break;
    }
    case WVA_SAT_ROUND_ROBIN:
        allocate_equally(c, un, n);
        break;
    default:
        break;
    }
}

/* greedy.go:35-104 */
void wvao_solve_greedy(const wva_fleet *f, wvao_alloc *cand, wvao_alloc *winners) {
    const int A = f->n_acc, S = f->n_servers;
    greedy_ctx c;
    c.f = f;
    c.cand = cand;
    c.winners = winners;
    c.available = (int *)malloc(sizeof(int) * (size_t)(f->n_types > 0 ? f->n_types : 1));
    for (int t = 0; t < f->n_types; t++) c.available[t] = f->type_capacity[t];

    greedy_entry *pool = (greedy_entry *)calloc((size_t)(S > 0 ? S : 1), sizeof(greedy_entry));
    greedy_entry **entries = (greedy_entry **)malloc(sizeof(void *) * (size_t)(S > 0 ? S : 1));
    greedy_entry **unalloc = (greedy_entry **)malloc(sizeof(void *) * (size_t)(S > 0 ? S : 1));
    int *alloc_ids = (int *)malloc(sizeof(int) * (size_t)(S * A > 0 ? S * A : 1));
    int n = 0;
    for (int s = 0; s < S; s++) {
        alloc_nil(&winners[s]); /* RemoveAllocation */
        int *ids = &alloc_ids[(size_t)s * A];
        int k = 0;
        for (int a = 0; a < A; a++)
            if (cand[(size_t)s * A + a].feasible) ids[k++] = a;
        if (k == 0) continue;
        /* stable insertion sort by value */
        for (int i = 1; i < k; i++) {
            int x = ids[i];
            int j = i - 1;
            while (j >= 0 && cmp_f32(cand[(size_t)s * A + ids[j]].value, cand[(size_t)s * A + x].value) > 0) {
                ids[j + 1] = ids[j];
                j--;
            }
            ids[j + 1] = x;
        }
        greedy_entry *e = &pool[n];
        e->server = s;
        e->priority = f->srv_priority[s];
        e->cur_index = 0;
        e->n_allocs = k;
        e->allocs = ids;
        if (k > 1)
            e->delta = cand[(size_t)s * A + ids[1]].value - cand[(size_t)s * A + ids[0]].value;
        else
            e->delta = FLT_MAX;
        entries[n] = e;
        n++;
    }
    sort_entries(&c, entries, n);

    if (f->delayed_best_effort) {
        int n_un = greedy_allocate(&c, entries, n, unalloc);
        best_effort(&c, unalloc, n_un);
    } else {
        /* the queue buffer is consumed in place, so copy each group out first */
        greedy_entry **group = (greedy_entry **)malloc(sizeof(void *) * (size_t)(n > 0 ? n : 1));
        int i = 0;
        while (i < n) {
            int j = i + 1;
            while (j < n && entries[j]->priority == entries[i]->priority) j++;
            int glen = j - i;
            memcpy(group, entries + i, sizeof(void *) * (size_t)glen);
            int n_un = greedy_allocate(&c, group, glen, unalloc);
            best_effort(&c, unalloc, n_un);
            i = j;
        }
        free(group);
    }
    free(alloc_ids);
    free(unalloc);
    free(entries);
    free(pool);
    free(c.available);
}

/* solver.go:32-59 */
void wvao_solve(const wva_fleet *f, wvao_alloc *cand, wvao_alloc *winners) {
    if (f->unlimited)
        wvao_solve_unlimited(f, cand, winners);
    else
        wvao_solve_greedy(f, cand, winners);
}

/* System.AllocateByType: pkg/core/system.go:271-300.  The reference walks s.Servers() (a Go map, random
 * order) and adds float32 costs as it goes; the order chosen here is ascending server index. */
void wvao_allocate_by_type(const wva_fleet *f, const wvao_alloc *winners, wvao_type_total *out) {
    for (int t = 0; t < f->n_types; ++t) {
        out[t].present = 0;
        out[t].limit = f->type_capacity[t]; /* s.capacity[nameType]: 0 when the map has no entry */
        out[t].count = 0;
        out[t].cost = 0.0f;
    }
    for (int s = 0; s < f->n_servers; ++s) {
        const wvao_alloc *al = &winners[s];
        if (!al->feasible) continue;                       /* serverAlloc == nil          :276-278 */
        if (al->acc < 0 || al->acc >= f->n_acc) continue;  /* s.accelerators[""] == nil   :282-284 */
        const int m = f->srv_model[s];
        if (m < 0 || m >= f->n_models) continue;           /* model == nil                :282-284 */
        const int t = f->acc_type[al->acc];
        if (t < 0 || t >= f->n_types) continue;
        out[t].present = 1;
        /* model.numInstances[accName] is a map lookup: 0 when the model has no profile on acc */
        const int64_t inst = f->perf_present[m * f->n_acc + al->acc] ? num_instances(f, m, al->acc) : 0;
        out[t].count += (int64_t)al->replicas * inst * (int64_t)f->acc_multiplicity[al->acc]; /* :296 */
        out[t].cost = out[t].cost + al->cost;                                                  /* :297 */
    }
}

/* CreateAllocationDiff (pkg/core/allocation.go:353-380) as Solver.Solve applies it (solver.go:51-58):
 * a = the server's current allocation (never nil: server.go:49), b = the solution's allocation. */
void wvao_allocation_diffs(const wva_fleet *f, const wvao_alloc *winners, wvao_diff *out) {
    for (int s = 0; s < f->n_servers; ++s) {
        const wvao_alloc *b = &winners[s];
        wvao_diff d;
        d.old_acc = f->srv_cur_acc[s];
        d.old_replicas = f->srv_cur_replicas[s];
        const float old_cost = f->srv_cur_cost[s];
        d.new_acc = WVA_ACC_ABSENT; /* "none" */
        d.new_replicas = 0;
        float new_cost = 0.0f;
        if (b->feasible) {
            d.new_acc = b->acc;
            d.new_replicas = b->replicas;
            new_cost = b->cost;
        }
        d.cost_diff = new_cost - old_cost;
        out[s] = d;
    }
}

/* ------------------------------------------------------------------------ */
/* candidate grid + latency sweep (the build's generalisation; SURVEY §8d)  */
/* ------------------------------------------------------------------------ */

/* Can (s, a) be analysed at all?  Mirrors the gates of CreateAllocation
 * (allocation.go:42-75) + the candidate-accelerator rule (server.go:70-82). */
static int pair_gate(const wva_fleet *f, int s, int a) {
    const int A = f->n_acc;
    if (!is_candidate_acc(f, s, a)) return 0;
    if (f->srv_arrival_rpm[s] < 0 || f->srv_in_tokens[s] < 0 || f->srv_out_tokens[s] < 0) return 0;
    int m = f->srv_model[s];
    if (m < 0 || m >= f->n_models) return 0;
    if (!f->perf_present[m * A + a]) return 0;
    if (!f->srv_has_target[s]) return 0;
    return 1;
}
static int zero_load(const wva_fleet *f, int s) {
    return f->srv_arrival_rpm[s] == 0 || f->srv_out_tokens[s] == 0;
}
static float total_rate_of(const wva_fleet *f, int s) { /* allocation.go:134-139 */
    if (f->srv_slo_tps[s] == 0) return f->srv_arrival_rpm[s] / 60;
    return f->srv_slo_tps[s] / (float)f->srv_out_tokens[s];
}

typedef struct cell_eval {
    int ok, feasible;
    wvao_metrics m;
    float ttft;
} cell_eval;

/* One grid cell: Analyze at totalRate/r with MaxBatchSize = b. */
static void eval_cell(const wva_fleet *f, int s, int a, int b, int r, cell_eval *ce) {
    const int A = f->n_acc;
    int m = f->srv_model[s];
    memset(ce, 0, sizeof(*ce));
    int max_queue;
    if (queue_states(b, f->tun.max_queue_to_batch_ratio, &max_queue) != 0) return;
    wvao_analyzer *qa = wvao_analyzer_new(b, max_queue, f->perf_alpha[m * A + a],
                                          f->perf_beta[m * A + a], f->perf_gamma[m * A + a],
                                          f->perf_delta[m * A + a], f->srv_in_tokens[s], f->srv_out_tokens[s]);
    if (!qa) return;
    float rate = total_rate_of(f, s) / (float)r;
    if (wvao_analyze(qa, rate, &ce->m) == 0) {
        ce->ok = 1;
        ce->ttft = ce->m.avg_wait_time + ce->m.avg_prefill_time;
        float slo_ttft = f->srv_slo_ttft[s], slo_itl = f->srv_slo_itl[s];
        int feas = (slo_ttft == 0 || ce->ttft <= slo_ttft) && (slo_itl == 0 || ce->m.avg_token_time <= slo_itl) &&
                   (r >= f->srv_min_replicas[s]);
        if (f->srv_slo_tps[s] > 0) { /* Size's stability margin, queueanalyzer.go:231-234 */
            float lambda_max = qa->rate_max / 1000;
            float lim = lambda_max * (1 - 0.1f);
            feas = feas && (rate / 1000 <= lim);
        }
        ce->feasible = feas;
    }
    wvao_analyzer_free(qa);
}

static int better(const wvao_alloc *x, const wvao_alloc *y) { /* x strictly better than y */
    if (x->value != y->value) return x->value < y->value;
    if (x->cost != y->cost) return x->cost < y->cost;
    if (x->replicas != y->replicas) return x->replicas < y->replicas;
    if (x->batch != y->batch) return x->batch < y->batch;
    return x->acc < y->acc;
}

void wvao_grid_solve(const wva_fleet *f, const wva_grid *g, wvao_cell *cells, wvao_alloc *winners) {
    const int A = f->n_acc, B = g->n_batch, R = g->n_replicas;
    g_solves = 0;
    g_states = 0;
    for (int s = 0; s < f->n_servers; s++) {
        wvao_alloc best;
        alloc_nil(&best);
        for (int a = 0; a < A; a++) {
            int gate = pair_gate(f, s, a);
            if (gate && zero_load(f, s)) {
                /* zero traffic: the reference's zeroLoadAllocation is the only candidate */
                wvao_alloc z;
                zero_load_allocation(f, s, f->srv_model[s], a, &z);
                z.value = wvao_transition_penalty(f->tun.accel_penalty_factor, f->srv_cur_acc[s],
                                                  f->srv_cur_replicas[s], f->srv_cur_cost[s], z.acc,
                                                  z.replicas, z.cost);
                if (!best.feasible || better(&z, &best)) best = z;
                gate = 0;
            }
            for (int bi = 0; bi < B; bi++) {
                for (int ri = 0; ri < R; ri++) {
                    size_t ci = (((size_t)s * A + a) * B + bi) * R + ri;
                    cell_eval ce;
                    memset(&ce, 0, sizeof(ce));
                    if (gate) eval_cell(f, s, a, g->batch[bi], g->replicas[ri], &ce);
                    if (cells) {
                        cells[ci].flags = (uint8_t)((ce.ok ? 1 : 0) | (ce.feasible ? 2 : 0));
                        cells[ci].ttft = ce.ok ? ce.ttft : 0;
                        cells[ci].itl = ce.ok ? ce.m.avg_token_time : 0;
                        cells[ci].rho = ce.ok ? ce.m.rho : 0;
                        cells[ci].throughput = ce.ok ? ce.m.throughput : 0;
                    }
                    if (ce.feasible) {
                        wvao_alloc c;
                        int r = g->replicas[ri];
                        int64_t total = (int64_t)num_instances(f, f->srv_model[s], a) * (int64_t)r;
                        c.feasible = 1;
                        c.acc = a;
                        c.replicas = r;
                        c.batch = g->batch[bi];
                        c.cost = f->acc_cost[a] * (float)total;
                        c.value = wvao_transition_penalty(f->tun.accel_penalty_factor, f->srv_cur_acc[s],
                                                          f->srv_cur_replicas[s], f->srv_cur_cost[s], a, r,
                                                          c.cost);
                        c.itl = ce.m.avg_token_time;
                        c.ttft = ce.ttft;
                        c.rho = ce.m.rho;
                        c.max_rate = ce.m.max_rate / 1000;
                        if (!best.feasible || better(&c, &best)) best = c;
                    }
                }
            }
        }
        winners[s] = best;
    }
}

void wvao_grid_cells(const wva_fleet *f, const wva_grid *g, int64_t c0, int64_t c1, wvao_cell *cells) {
    const int A = f->n_acc, B = g->n_batch, R = g->n_replicas;
    g_solves = 0;
    g_states = 0;
    for (int64_t ci = c0; ci < c1; ci++) {
        int ri = (int)(ci % R);
        int bi = (int)((ci / R) % B);
        int a = (int)((ci / ((int64_t)R * B)) % A);
        int s = (int)(ci / ((int64_t)R * B * A));
        cell_eval ce;
        memset(&ce, 0, sizeof(ce));
        if (pair_gate(f, s, a) && !zero_load(f, s)) eval_cell(f, s, a, g->batch[bi], g->replicas[ri], &ce);
        wvao_cell *o = &cells[ci - c0];
        o->flags = (uint8_t)((ce.ok ? 1 : 0) | (ce.feasible ? 2 : 0));
        o->ttft = ce.ok ? ce.ttft : 0;
        o->itl = ce.ok ? ce.m.avg_token_time : 0;
        o->rho = ce.ok ? ce.m.rho : 0;
        o->throughput = ce.ok ? ce.m.throughput : 0;
    }
}

/* Batch size a (server, accelerator) pair is analysed at outside the grid:
 * allocation.go:77-87. */
static int64_t pair_batch(const wva_fleet *f, int s, int a) {
    const int A = f->n_acc;
    int m = f->srv_model[s];
    if (f->srv_max_batch[s] > 0) return f->srv_max_batch[s];
    int64_t t = (int64_t)f->perf_max_batch[m * A + a] * (int64_t)f->perf_at_tokens[m * A + a] /
                f->srv_out_tokens[s];
    return t > 1 ? t : 1;
}

void wvao_sweep(const wva_fleet *f, int n_rates, uint8_t *valid, float *rate, float *ttft, float *itl,
                float *throughput, float *rho) {
    const int A = f->n_acc;
    g_solves = 0;
    g_states = 0;
    for (int s = 0; s < f->n_servers; s++) {
        for (int a = 0; a < A; a++) {
            size_t base = ((size_t)s * A + a) * (size_t)n_rates;
            wvao_analyzer *qa = NULL;
            /* the sweep ignores keepAccelerator: it characterises every profile */
            int gate = f->srv_in_tokens[s] >= 0 && f->srv_out_tokens[s] >= 1 && f->srv_model[s] >= 0 &&
                       f->srv_model[s] < f->n_models && f->perf_present[f->srv_model[s] * A + a];
            int max_queue;
            int64_t N = gate ? pair_batch(f, s, a) : 0;
            if (gate && queue_states(N, f->tun.max_queue_to_batch_ratio, &max_queue) == 0) {
                int m = f->srv_model[s];
                qa = wvao_analyzer_new((int)N, max_queue, f->perf_alpha[m * A + a],
                                       f->perf_beta[m * A + a], f->perf_gamma[m * A + a],
                                       f->perf_delta[m * A + a], f->srv_in_tokens[s], f->srv_out_tokens[s]);
            }
            for (int i = 0; i < n_rates; i++) {
                valid[base + i] = 0;
                rate[base + i] = ttft[base + i] = itl[base + i] = throughput[base + i] = rho[base + i] = 0;
            }
            if (!qa) continue;
            float lo = qa->rate_min;
            float hi = qa->rate_max * 0.999f;
            float span = hi - lo;
            for (int i = 0; i < n_rates; i++) {
                float frac = n_rates > 1 ? (float)i / (float)(n_rates - 1) : 0.0f;
                float step = span * frac;
                float rt = lo + step;
                rate[base + i] = rt;
                wvao_metrics mt;
                /* every sweep point is a fresh model (no stale p[0]) */
                memset(qa->p, 0, sizeof(double) * ((size_t)qa->K + 1));
                if (wvao_analyze(qa, rt, &mt) == 0) {
                    valid[base + i] = 1;
                    ttft[base + i] = mt.avg_wait_time + mt.avg_prefill_time;
                    itl[base + i] = mt.avg_token_time;
                    throughput[base + i] = mt.throughput;
                    rho[base + i] = mt.rho;
                }
            }
            wvao_analyzer_free(qa);
        }
    }
}

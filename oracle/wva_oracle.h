/*
 * wva_oracle.h — CPU restatement of the WVA optimizer hot path (TEST INFRASTRUCTURE).
 *
 * This is the parity oracle (SURVEY.md §8c).  It is NOT part of the product: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load it.  The product (workload_variant_autoscaler_b200/csrc) never links
 * or calls anything in this directory.
 *
 * Semantics restated: Go 1.23 on amd64, GOAMD64=v1 — IEEE binary32/64, RNE, no FMA
 * fusion, `a*b/c` = `(a*b)/c`, builtin min/max propagate NaN.  Build with
 * `-O2 -ffp-contract=off -fno-fast-math` (see oracle/Makefile).
 *
 * Pinning status: every known-answer value the reference's own tests hold for
 * this path is reproduced (tests/test_oracle_kat.py); float outputs under non-zero
 * load are pinned by no reference test (SURVEY.md §4), so beyond those KATs the
 * oracle is cross-checked by an independent numpy restatement
 * (oracle/restate_np.py).  The Go reference itself cannot be run here (no Go
 * toolchain): "parity pinned to the reference's KATs; float values under load
 * pinned to the restatement only".
 */
#ifndef WVA_ORACLE_H
#define WVA_ORACLE_H

#include <stdint.h>

#include "../include/wva_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* pkg/analyzer/queueanalyzer.go:61-70 */
typedef struct wvao_metrics {
    float throughput;
    float avg_resp_time;
    float avg_wait_time;
    float avg_num_in_serv;
    float avg_prefill_time;
    float avg_token_time;
    float max_rate;
    float rho;
} wvao_metrics;

/* pkg/analyzer/queueanalyzer.go:73-84 */
typedef struct wvao_target_perf {
    float ttft, itl, tps;
} wvao_target_perf;
typedef struct wvao_target_rate {
    float rate_ttft, rate_itl, rate_tps;
} wvao_target_rate;

/* raw model statistics (pkg/analyzer/queuemodel.go:10-19, mm1kmodel.go:10-16) */
typedef struct wvao_model_stats {
    int32_t is_valid;
    float lambda, mu, rho;
    float avg_resp_time, avg_wait_time, avg_serv_time, avg_num_in_system, avg_queue_length;
    float throughput, avg_num_in_servers;
    double sum_p;
} wvao_model_stats;

typedef struct wvao_analyzer wvao_analyzer; /* QueueAnalyzer + its MM1ModelStateDependent */
typedef struct wvao_mm1k wvao_mm1k;         /* MM1KModel (closed form; off the production path) */

/* ---- pkg/analyzer ------------------------------------------------------- */
float wvao_prefill_time(float gamma, float delta, int in_tokens, float batch); /* queueanalyzer.go:257-262 */
float wvao_decode_time(float alpha, float beta, float batch);                  /* :264-266 */
float wvao_effective_concurrency(float avg_serv_time, float alpha, float beta, float gamma,
                                 float delta, int in_tokens, int out_tokens,
                                 int max_batch); /* :296-302 */
int wvao_within_tolerance(float x, float value, float tol); /* utils.go:12-20 */

/* utils.go:26-70. eval returns 0 on success (y in *y), non-zero = error.
 * Returns 0 ok, 1 invalid range, 2 eval error. */
typedef int (*wvao_eval_fn)(void *ctx, float x, float *y);
int wvao_binary_search(float xmin, float xmax, float ytarget, wvao_eval_fn eval, void *ctx,
                       float *xstar, int *ind);

/* MM1KModel: mm1kmodel.go:19-92 */
wvao_mm1k *wvao_mm1k_new(int K);
void wvao_mm1k_free(wvao_mm1k *m);
void wvao_mm1k_solve(wvao_mm1k *m, float lambda, float mu, wvao_model_stats *out);
const double *wvao_mm1k_probs(const wvao_mm1k *m);
/* math.Pow(x, n) for an integer n >= 0 as the Go standard library computes it (src/math/pow.go) */
double wvao_go_pow_uint(double x, int64_t n);

/* NewQueueAnalyzer / BuildModel: queueanalyzer.go:87-131. NULL on check() failure. */
wvao_analyzer *wvao_analyzer_new(int max_batch, int max_queue, float alpha, float beta, float gamma,
                                 float delta, int in_tokens, int out_tokens);
wvao_analyzer *wvao_model_new_rates(int K, const float *serv_rate, int n); /* NewMM1ModelStateDependent :16-24 */
void wvao_analyzer_free(wvao_analyzer *qa);
void wvao_analyzer_rate_range(const wvao_analyzer *qa, float *rmin, float *rmax);
const float *wvao_analyzer_serv_rate(const wvao_analyzer *qa); /* [max_batch] */
const double *wvao_analyzer_probs(const wvao_analyzer *qa);    /* [K+1] after a solve */
int wvao_analyzer_K(const wvao_analyzer *qa);
/* Model.Solve(lambda, mu) on the state-dependent model: queuemodel.go:27-37 */
void wvao_model_solve(wvao_analyzer *qa, float lambda, float mu, wvao_model_stats *out);
/* Analyze: queueanalyzer.go:134-174. 0 ok; 1 rate<=0; 2 rate>max; 3 invalid model */
int wvao_analyze(wvao_analyzer *qa, float request_rate, wvao_metrics *out);
/* Size: :185-255. 0 ok, non-zero error (1 bad target, 2 ttft search, 3 itl search, 4 analyze) */
int wvao_size(wvao_analyzer *qa, const wvao_target_perf *target, wvao_target_rate *rates,
              wvao_metrics *metrics, wvao_target_perf *achieved);
int wvao_eval_ttft(wvao_analyzer *qa, float x, float *y); /* :270-279 */
int wvao_eval_itl(wvao_analyzer *qa, float x, float *y);  /* :283-290 */
/* number of Model.Solve calls made on this analyzer so far (instrumentation) */
int64_t wvao_analyzer_solves(const wvao_analyzer *qa);

/* ---- pkg/core ----------------------------------------------------------- */
/* one candidate record = core.Allocation (allocation.go:13-24) */
typedef struct wvao_alloc {
    int32_t feasible;
    int32_t acc;
    int32_t replicas;
    int32_t batch;
    float cost, value, itl, ttft, rho, max_rate;
} wvao_alloc;

/* CreateAllocation(server, acc): allocation.go:27-163 (value = cost). */
void wvao_create_allocation(const wva_fleet *f, int s, int a, wvao_alloc *out);
/* TransitionPenalty: allocation.go:291-300 */
float wvao_transition_penalty(float factor, int cur_acc, int cur_replicas, float cur_cost,
                              int new_acc, int new_replicas, float new_cost);
/* Server.Calculate for all servers: server.go:55-82. out[S*A]. */
void wvao_calculate(const wva_fleet *f, wvao_alloc *out);
/* solves performed by the last wvao_calculate / wvao_grid call (instrumentation) */
int64_t wvao_last_solves(void);
int64_t wvao_last_states(void);
/* Queue models refused since the previous call, and reset to 0: a model of N + N * max_queue_to_batch_ratio
 * >= 2^31 states (computed in 64 bits, as Go's int) is outside the int32 domain of this oracle and of the CUDA
 * library.  Its candidate, cell or sweep points are left nil / invalid; callers treat a non-zero count as
 * "unsupported" (the library returns WVA_ERR_UNSUPPORTED for such a call). */
int64_t wvao_take_unsupported(void);

/* ---- pkg/solver --------------------------------------------------------- */
/* SolveUnlimited: solver.go:63-79, deterministic tie-break = lowest acc id. */
void wvao_solve_unlimited(const wva_fleet *f, const wvao_alloc *cand, wvao_alloc *winners);
/* SolveGreedy: greedy.go:35-341 (stable sorts; ties by server id / acc id). `cand` is
 * modified by the best-effort policies exactly as the reference mutates allocations. */
void wvao_solve_greedy(const wva_fleet *f, wvao_alloc *cand, wvao_alloc *winners);
/* Solver.Solve: dispatch on f->unlimited. */
void wvao_solve(const wva_fleet *f, wvao_alloc *cand, wvao_alloc *winners);

/* ---- pkg/core/system.go:271-300, pkg/core/allocation.go:353-380 --------------------------- */
typedef struct wvao_type_total { /* core.AllocationByType */
    int32_t present;           /* the type has an entry in allocationByType */
    int32_t limit;             /* s.capacity[type] */
    int64_t count;
    float cost;
} wvao_type_total;
/* System.AllocateByType over the solution `winners` [S] -> out [T]; float32 cost summed in ascending
 * server index (the reference iterates a Go map, i.e. in random order). */
void wvao_allocate_by_type(const wva_fleet *f, const wvao_alloc *winners, wvao_type_total *out);
typedef struct wvao_diff { /* core.AllocationDiff */
    int32_t old_acc, new_acc, old_replicas, new_replicas;
    float cost_diff;
} wvao_diff;
/* CreateAllocationDiff(server.CurAllocation(), server.Allocation()) for every server (solver.go:51-58). */
void wvao_allocation_diffs(const wva_fleet *f, const wvao_alloc *winners, wvao_diff *out);

/* ---- grid / sweep (build's generalisation, SURVEY.md §8d) --------------- */
typedef struct wvao_cell {
    uint8_t flags; /* bit0 analyze ok, bit1 SLO feasible */
    float ttft, itl, rho, throughput;
} wvao_cell;
/* cells may be NULL; winners[S]. */
void wvao_grid_solve(const wva_fleet *f, const wva_grid *g, wvao_cell *cells, wvao_alloc *winners);
/* evaluate a contiguous range of cells [c0, c1) only (bounded CPU baseline sample) */
void wvao_grid_cells(const wva_fleet *f, const wva_grid *g, int64_t c0, int64_t c1, wvao_cell *cells);
void wvao_sweep(const wva_fleet *f, int n_rates, uint8_t *valid, float *rate, float *ttft,
                float *itl, float *throughput, float *rho);

#ifdef __cplusplus
}
#endif
#endif

/*
 * wva_b200.h — C ABI of the H100-native WVA optimizer hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b): the seam between WVA's L2
 * adapters (internal/modelanalyzer, internal/optimizer) and the L1 "inferno"
 * optimizer library (pkg/analyzer, pkg/core, pkg/solver, pkg/manager).  The Go
 * side packs a `config.SystemSpec` (pkg/config/types.go:11-21) into the flat
 * SoA `wva_fleet` below, makes ONE call, and reads back what
 * `System.GenerateSolution()` (pkg/core/system.go:303-319) would have produced.
 *
 * Plain C: pointers + sizes only.  All arrays are caller-owned HOST memory; the
 * library never retains a caller pointer after a call returns (cgo rule).  One
 * call at a time per handle (the reference L1 is non-reentrant as well:
 * pkg/core/system.go:10-13, pkg/analyzer/utils.go:73).
 *
 * Error model (pkg/core/allocation.go:42-70,111-130,150-153): an infeasible
 * candidate is DATA (`feasible == 0`, the reference's `nil *Allocation`), never
 * an error code.  Negative return values are hard errors only (bad arguments,
 * CUDA failure, missing device).
 *
 * Arithmetic contract: results are bit-identical to the reference Go code built
 * for amd64 at GOAMD64=v1 (IEEE binary32/binary64, round-to-nearest-even, no FMA
 * contraction) — integers exactly, float32 outputs bit-for-bit.
 */
#ifndef WVA_B200_H
#define WVA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WVA_ABI_VERSION 2

/* ---- return codes ------------------------------------------------------- */
#define WVA_OK 0
#define WVA_ERR_BAD_ARG (-1)     /* NULL pointer, negative size, id out of range   */
#define WVA_ERR_NO_DEVICE (-2)   /* no CUDA device / requested ordinal missing      */
#define WVA_ERR_CUDA (-3)        /* a CUDA runtime call failed (see wva_last_error) */
#define WVA_ERR_NOMEM (-4)       /* host or device allocation failed                */
#define WVA_ERR_STATE (-5)       /* call sequence error (e.g. resolve before upload)*/
#define WVA_ERR_UNSUPPORTED (-6) /* input outside the supported numeric domain      */

/* ---- sentinels ---------------------------------------------------------- */
#define WVA_ACC_NONE (-1)    /* accelerator name "" (pkg/core/allocation.go:264)    */
#define WVA_ACC_UNKNOWN (-2) /* a name that is not in the accelerator table         */
#define WVA_ACC_ABSENT (-3)  /* no allocation at all: CreateAllocationDiff's "none"  */

/* saturation policies: pkg/config/config.go:4-41 */
#define WVA_SAT_NONE 0
#define WVA_SAT_PRIORITY_EXHAUSTIVE 1
#define WVA_SAT_PRIORITY_ROUND_ROBIN 2
#define WVA_SAT_ROUND_ROBIN 3

typedef struct wva_handle wva_handle;

/*
 * Tunables that are package-level variables in the reference
 * (pkg/config/defaults.go:18,21).  wva_tunables_default() fills the reference values.
 */
typedef struct wva_tunables {
    int32_t max_queue_to_batch_ratio; /* config.MaxQueueToBatchRatio = 10          */
    float accel_penalty_factor;       /* config.AccelPenaltyFactor   = 0.1         */
} wva_tunables;

/*
 * The fleet: flat SoA image of config.SystemSpec after the joins that
 * System.SetFromSpec (pkg/core/system.go:82-194) performs with Go maps.
 *
 *   A accelerators   — config.AcceleratorSpec   (pkg/config/types.go:29-37)
 *   T accelerator types + capacity — config.AcceleratorCount (types.go:52-56)
 *   M models; perf data per (model, accelerator), row-major [M*A]
 *                    — config.ModelAcceleratorPerfData (types.go:64-72)
 *   S servers        — config.ServerSpec (types.go:112-121) joined with its
 *                      service class / model target (types.go:92-105)
 */
typedef struct wva_fleet {
    /* accelerators [A] */
    int32_t n_acc;
    const float *acc_cost;           /* AcceleratorSpec.Cost (cents/hr)                 */
    const int32_t *acc_multiplicity; /* AcceleratorSpec.Multiplicity                    */
    const int32_t *acc_type;         /* type id in [0, n_types)                         */

    /* accelerator types [T]; only read in limited (greedy) mode */
    int32_t n_types;
    const int32_t *type_capacity; /* CapacityData count; types absent in Go map = 0  */

    /* per (model, accelerator) [M*A], index m*A + a */
    int32_t n_models;
    const uint8_t *perf_present;   /* 1 iff model.PerfData(acc) != nil                */
    const float *perf_alpha;       /* DecodeParms.Alpha                               */
    const float *perf_beta;        /* DecodeParms.Beta                                */
    const float *perf_gamma;       /* PrefillParms.Gamma                              */
    const float *perf_delta;       /* PrefillParms.Delta                              */
    const int32_t *perf_acc_count; /* AccCount (<=0 -> 1, pkg/core/model.go:52-55)    */
    const int32_t *perf_max_batch; /* MaxBatchSize                                    */
    const int32_t *perf_at_tokens; /* AtTokens                                        */

    /* servers [S] */
    int32_t n_servers;
    const int32_t *srv_model;       /* model id, or -1 if the model name is unknown   */
    const int32_t *srv_priority;    /* service class priority (server.go:92-97)       */
    const uint8_t *srv_has_target;  /* service class exists AND has a target for model*/
    const float *srv_slo_itl;       /* Target.ITL  (msec)                             */
    const float *srv_slo_ttft;      /* Target.TTFT (msec)                             */
    const float *srv_slo_tps;       /* Target.TPS  (tokens/sec)                       */
    const uint8_t *srv_keep_acc;    /* ServerSpec.KeepAccelerator                     */
    const int32_t *srv_min_replicas;/* ServerSpec.MinNumReplicas                      */
    const int32_t *srv_max_batch;   /* ServerSpec.MaxBatchSize override (0 = none)    */
    const float *srv_arrival_rpm;   /* ServerLoadSpec.ArrivalRate (req/min)           */
    const int32_t *srv_in_tokens;   /* ServerLoadSpec.AvgInTokens                     */
    const int32_t *srv_out_tokens;  /* ServerLoadSpec.AvgOutTokens                    */
    const int32_t *srv_cur_acc;     /* CurrentAlloc.Accelerator: id, NONE or UNKNOWN  */
    const int32_t *srv_cur_replicas;/* CurrentAlloc.NumReplicas                       */
    const float *srv_cur_cost;      /* CurrentAlloc.Cost                              */

    /* optimizer spec (pkg/config/types.go:151-155) */
    uint8_t unlimited;
    uint8_t delayed_best_effort;
    int32_t saturation_policy; /* WVA_SAT_* */

    wva_tunables tun;
} wva_fleet;

/*
 * One candidate allocation per (server, accelerator): the fields of
 * core.Allocation (pkg/core/allocation.go:13-24).  Arrays have S*A entries
 * (index s*A + a) for candidate tables, S entries for per-server winners.
 * Any pointer may be NULL (that column is not written).
 */
typedef struct wva_allocs {
    uint8_t *feasible;  /* 0 = nil allocation                                        */
    int32_t *acc;       /* accelerator id; WVA_ACC_NONE for the zero-replica case    */
    int32_t *replicas;  /* numReplicas                                               */
    int32_t *batch;     /* batchSize                                                 */
    float *cost;        /* cost                                                      */
    float *value;       /* value (transition penalty, pkg/core/server.go:60-63)      */
    float *itl;         /* expected inter-token latency (msec)                       */
    float *ttft;        /* expected queueing + prefill time (msec)                   */
    float *rho;         /* utilisation                                               */
    float *max_rate;    /* maxArrvRatePerReplica (req/msec)                          */
} wva_allocs;

/*
 * Candidate grid (the build's generalisation, SURVEY.md §8d): every
 * (server, accelerator, batch, replica) cell is one QueueAnalyzer.Analyze
 * (pkg/analyzer/queueanalyzer.go:134-174) at rate totalRate(server)/replicas
 * with MaxBatchSize = batch, followed by the SLO feasibility test, the cost and
 * the transition penalty.  Cell index = ((s*A + a)*B + bi)*R + ri.
 */
typedef struct wva_grid {
    int32_t n_batch;
    const int32_t *batch; /* [B] batch sizes, each >= 1                           */
    int32_t n_replicas;
    const int32_t *replicas; /* [R] replica counts, each >= 1                     */
} wva_grid;

/* Optional per-cell table (any pointer may be NULL). flags bit0 = Analyze ok,
 * bit1 = SLO-feasible (implies bit0). */
typedef struct wva_cells {
    uint8_t *flags;
    float *ttft;       /* AvgWaitTime + AvgPrefillTime                             */
    float *itl;        /* AvgTokenTime                                             */
    float *rho;        /* Rho                                                      */
    float *throughput; /* Throughput (req/sec)                                     */
} wva_cells;

/* Latency sweep (BASELINE config 3): for each (server, accelerator) pair,
 * Analyze at n_rates rates linearly spaced in [RateRange.Min, RateRange.Max*0.999].
 * Output index = (s*A + a)*n_rates + i. valid = 0 where the pair has no model or
 * Analyze returned an error. */
typedef struct wva_sweep_out {
    uint8_t *valid;
    float *rate;       /* req/sec                                                  */
    float *ttft;
    float *itl;
    float *throughput;
    float *rho;
} wva_sweep_out;

/* ---- lifecycle ---------------------------------------------------------- */

/* Reference values of the package-level tunables. */
void wva_tunables_default(wva_tunables *t);

/* Create an engine bound to CUDA device `device` (ordinal). Fails with
 * WVA_ERR_NO_DEVICE when there is no such GPU: there is no CPU fallback. */
int wva_create(wva_handle **out, int device);
void wva_destroy(wva_handle *h);

const char *wva_strerror(int code);
/* Text of the last hard error on this handle ("" if none). */
const char *wva_last_error(const wva_handle *h);
int wva_abi_version(void);

/* ---- the hot path -------------------------------------------------------- */

/*
 * Server.Calculate for every server (pkg/core/server.go:55-67): one
 * CreateAllocation (pkg/core/allocation.go:27-163) per candidate accelerator and
 * value = TransitionPenalty(current, candidate) (allocation.go:291-300).
 * Replaces ModelAnalyzer.AnalyzeModel (internal/modelanalyzer/analyzer.go:25-34)
 * called in a loop at internal/controller/variantautoscaling_controller.go:149-156.
 * `candidates` has S*A entries.
 *
 * Queue sizes (wva_analyze, wva_solve, wva_resolve and every call below that builds queue models): a load pair,
 * i.e. one that passes the gates with a positive arrival rate and out_tokens >= 1, builds the reference's queue
 * model of batch size N (srv_max_batch, else max(perf_max_batch * perf_at_tokens / out_tokens, 1)) with
 * N + N * max_queue_to_batch_ratio states.  Both are computed in 64 bits, as Go's int.  The call returns
 * WVA_ERR_UNSUPPORTED, before any kernel is launched and with a wva_last_error text naming the cause, when such
 * an N is above 2^20 or such a model has 2^31 states or more: the reference would need a p[] vector of 2^31
 * doubles or more, and this library counts states in int32.  Zero-load pairs (zeroLoadAllocation reads
 * perf_max_batch directly) and gated pairs build no model and are never refused.  wva_resolve applies the rule to
 * the resident fleet as wva_update_load left it.
 */
int wva_analyze(wva_handle *h, const wva_fleet *fleet, wva_allocs *candidates);

/*
 * Analyze + Solver.Solve (pkg/solver/solver.go:32-59): SolveUnlimited
 * (solver.go:63-79) when fleet->unlimited, else SolveGreedy
 * (pkg/solver/greedy.go:35-104) over the device-computed candidates.  Replaces
 * VariantAutoscalingsEngine.Optimize (internal/optimizer/optimizer.go:30-54) =
 * Manager.Optimize (pkg/manager/manager.go:21-27) + System.GenerateSolution
 * (pkg/core/system.go:303-319).  `winners` has S entries; `candidates` (S*A) may
 * be NULL.  Ties on value are resolved to the lowest accelerator id (the
 * reference resolves them by Go map iteration order, i.e. randomly).
 */
int wva_solve(wva_handle *h, const wva_fleet *fleet, wva_allocs *candidates,
              wva_allocs *winners);

/*
 * Full candidate grid + per-server min-value SLO-feasible cell.
 * Winner order: value, then cost, then replicas, then batch, then accelerator id
 * (all ascending).  `cells` may be NULL.  WVA_ERR_UNSUPPORTED (the queue-size rule of wva_analyze, for
 * wva_grid_solve_device too): some server has a load pair, the grid has a replica level, and the largest listed
 * batch size b has b * (1 + max_queue_to_batch_ratio) >= 2^31.
 */
int wva_grid_solve(wva_handle *h, const wva_fleet *fleet, const wva_grid *grid,
                   wva_cells *cells, wva_allocs *winners);

/*
 * Size grid: Server.Calculate (the reference's CreateAllocation rule, as in wva_analyze) once per listed
 * batch size, and the min-value (accelerator, batch size) per server.
 *
 * Candidate (s, a, bi), index (s*A + a)*n_batch + bi, is exactly what wva_analyze returns for (s, a) on the
 * same fleet with every server's srv_max_batch set to batch[bi]: N = batch[bi], the queue size is
 * max_queue_to_batch_ratio * N, and a zero-load candidate uses N in zeroLoadAllocation.  perf_max_batch,
 * perf_at_tokens and srv_max_batch are not read.  The candidate rule (keepAccelerator), the gates and
 * value = TransitionPenalty(current, candidate) are those of wva_analyze.
 *
 * winners[s] is the feasible candidate of server s with the smallest value under SolveUnlimited's rule
 * (strict '<' starting from MaxFloat32: a NaN value, or one not below MaxFloat32, never wins); ties go to
 * the smaller batch size, then the lower accelerator id.  With one batch size this is wva_solve's winner.
 * Repeated batch sizes give identical records.  Like wva_grid_solve, the minimum does not read
 * fleet->unlimited or the capacities.  The winners stay resident for wva_summarize.
 *
 * `candidates` (S*A*n_batch entries) may be NULL; `winners` has S entries.  n_batch == 0 is valid (every
 * winner is nil).  WVA_ERR_BAD_ARG: n_batch < 0, batch NULL with n_batch > 0, or a batch size outside
 * [1, 2^20].  WVA_ERR_UNSUPPORTED: S*A*n_batch >= 2^31; some server has a load pair and the largest listed
 * batch size b has b * (1 + max_queue_to_batch_ratio) >= 2^31 (the queue-size rule of wva_analyze); or, as for
 * wva_solve, too many candidates need the stored-vector fallback or its rescale loop would not terminate.
 */
int wva_size_grid(wva_handle *h, const wva_fleet *fleet, int32_t n_batch, const int32_t *batch,
                  wva_allocs *candidates, wva_allocs *winners);

/*
 * Load grid: Server.Calculate (as in wva_analyze) and SolveUnlimited's winner at each of n_levels caller-given
 * arrival-rate rows, e.g. a load forecast or a peak scenario.
 *
 * Let f_l be the fleet with srv_arrival_rpm replaced by row l of arrival_rpm ([n_levels * S], index l*S + s,
 * req/min).  Candidate block l (records (l*S + s)*A + a) is byte for byte what wva_analyze returns for f_l,
 * value = TransitionPenalty included.  Winner block l (records l*S + s) is wva_solve's winner block for f_l with
 * unlimited = 1: strict '<' from MaxFloat32, ties to the lower accelerator id.  Per level a pair is nil at a
 * negative rate, zeroLoadAllocation at rate 0 (or out_tokens 0), and sized under load otherwise, NaN and +Inf
 * included.  fleet->srv_arrival_rpm, fleet->unlimited and the capacities are not read; every other column
 * (tokens, targets, current allocations) comes from `fleet`.  Each candidate block is a valid input for
 * wva_solve_greedy, which serves limited mode.
 *
 * The sizing part of CreateAllocation (QueueAnalyzer.Size and rateStar) does not read the load, so it runs once
 * per (server, accelerator); only the replica count, the cost and one Analyze run per level.
 *
 * The fleet becomes resident, as with every call that takes one; there is no single solution afterwards, so
 * wva_summarize returns WVA_ERR_STATE.  `candidates` (n_levels*S*A entries) may be NULL; `winners` has
 * n_levels*S entries.  n_levels == 0 is valid (nothing is written).  WVA_ERR_BAD_ARG: n_levels < 0,
 * arrival_rpm NULL with n_levels > 0, or winners NULL.  WVA_ERR_UNSUPPORTED: S*A*n_levels >= 2^31 (refused
 * before the fleet is read), or a level on which wva_analyze of f_l fails the same way (a NaN rate whose
 * rescale loop would not terminate, too many stored-vector fallbacks, a load pair outside wva_analyze's
 * queue-size rule).
 */
int wva_load_grid(wva_handle *h, const wva_fleet *fleet, int32_t n_levels, const float *arrival_rpm,
                  wva_allocs *candidates, wva_allocs *winners);

/*
 * SLO grid: Server.Calculate (as in wva_analyze) and SolveUnlimited's winner at each of n_levels caller-given
 * rows of service-class targets, e.g. candidate ITL / TTFT / TPS targets before they are chosen.
 *
 * Let f_l be the fleet with srv_slo_itl, srv_slo_ttft and srv_slo_tps replaced by row l of slo_itl, slo_ttft and
 * slo_tps (each [n_levels * S], index l*S + s, in the units of the fleet's columns).  Candidate block l (records
 * (l*S + s)*A + a) is byte for byte what wva_analyze returns for f_l, value = TransitionPenalty included.  Winner
 * block l (records l*S + s) is wva_solve's winner block for f_l with unlimited = 1: strict '<' from MaxFloat32,
 * ties to the lower accelerator id.  fleet->srv_slo_*, fleet->unlimited and the capacities are not read; every
 * other column comes from `fleet`, and srv_has_target still gates (a server without a target is nil at every
 * level).  Each candidate block is a valid input for wva_solve_greedy, which serves limited mode.
 *
 * Deduplication: each bisection of QueueAnalyzer.Size reads exactly one target (the TTFT search TargetTTFT, the
 * ITL search TargetITL) and nothing else of the service class, so a search is determined by (server, accelerator,
 * which search, target bits).  Each distinct (server, search, target) that some level needs runs once per
 * (server, accelerator); a level needs it when its three targets are not negative and the target is > 0 (0, -0
 * and NaN disable a search).  Only lambda*, rateStar, the replica count, the cost and two Analyze calls run per
 * level: an 8 x 8 ITL x TTFT grid runs 16 searches per pair instead of 128.
 *
 * The fleet becomes resident, as with every call that takes one; there is no single solution afterwards, so
 * wva_summarize returns WVA_ERR_STATE.  `candidates` (n_levels*S*A entries) may be NULL; `winners` has
 * n_levels*S entries.  n_levels == 0 is valid (nothing is written).  WVA_ERR_BAD_ARG: n_levels < 0, a row list
 * NULL with n_levels * S > 0, or winners NULL.  WVA_ERR_UNSUPPORTED: S*A*n_levels >= 2^31 (refused before the
 * fleet is read); 2^31 or more search records (distinct keys x A); a load pair outside wva_analyze's queue-size
 * rule (with n_levels > 0); or exactly the levels on which wva_analyze of f_l fails the same way (a rescale loop
 * that would not terminate, which a NaN or tiny TPS target can cause, or too many stored-vector fallbacks).  A
 * search that no level's reference would run (the ITL search after a failed TTFT search) does not fail the call.
 */
int wva_slo_grid(wva_handle *h, const wva_fleet *fleet, int32_t n_levels, const float *slo_itl,
                 const float *slo_ttft, const float *slo_tps, wva_allocs *candidates, wva_allocs *winners);

/*
 * Workload grid: Server.Calculate (as in wva_analyze) and SolveUnlimited's winner at each of n_levels caller-given
 * rows of (arrival rate, average input tokens, average output tokens), e.g. a forecast in which prompts or answers
 * grow, or a daily mix of chat and batch traffic.
 *
 * Let f_l be the fleet with srv_arrival_rpm, srv_in_tokens and srv_out_tokens replaced by row l of arrival_rpm
 * (req/min), in_tokens and out_tokens (each [n_levels * S], index l*S + s).  Candidate block l (records
 * (l*S + s)*A + a) is byte for byte what wva_analyze returns for f_l, value = TransitionPenalty included.  Winner
 * block l (records l*S + s) is wva_solve's winner block for f_l with unlimited = 1: strict '<' from MaxFloat32,
 * ties to the lower accelerator id.  Per level a pair is nil at a negative rate or negative tokens,
 * zeroLoadAllocation at rate 0 or out_tokens 0, and sized under load otherwise, NaN and +Inf rates included.
 * fleet->srv_arrival_rpm, srv_in_tokens, srv_out_tokens, fleet->unlimited and the capacities are not read; every
 * other column comes from `fleet`.  Each candidate block is a valid input for wva_solve_greedy, which serves
 * limited mode.
 *
 * Deduplication: QueueAnalyzer.Size, lambda* and rateStar read a server's tokens but not its rate, so they run
 * once per (server, accelerator, in_tokens, out_tokens) that some level uses under load (DESIGN.md §3.12).  Only
 * the replica count, the cost and one Analyze run per level.  With the fleet's own tokens on every row the call
 * sizes what wva_load_grid sizes, and returns the same bytes.
 *
 * The fleet becomes resident, as with every call that takes one; there is no single solution afterwards, so
 * wva_summarize returns WVA_ERR_STATE.  `candidates` (n_levels*S*A entries) may be NULL; `winners` has
 * n_levels*S entries.  n_levels == 0 is valid (nothing is written).  WVA_ERR_BAD_ARG: n_levels < 0, a row list
 * NULL with n_levels * S > 0, or winners NULL.  WVA_ERR_UNSUPPORTED: S*A*n_levels >= 2^31 (refused before the
 * fleet is read; the distinct keys x A are then below 2^31 as well), or exactly the levels on which wva_analyze of
 * f_l fails the same way: a load pair outside the queue-size rule (its batch size comes from that level's
 * out_tokens, so a small out_tokens can push it above 2^20), a rescale loop that would not terminate, or too many
 * stored-vector fallbacks.  A token pair that no level uses under load (its levels all have rate 0, a negative
 * rate or out_tokens 0) is never sized and does not fail the call.
 */
int wva_workload_grid(wva_handle *h, const wva_fleet *fleet, int32_t n_levels, const float *arrival_rpm,
                      const int32_t *in_tokens, const int32_t *out_tokens, wva_allocs *candidates,
                      wva_allocs *winners);

/*
 * Workload trace: the reference's reconcile replayed over n_ticks caller-given rows of (arrival rate, average input
 * tokens, average output tokens), each tick's winner becoming the next tick's current allocation, e.g. what the
 * autoscaler does over a recorded day or a forecast, and what it costs.  The rows are laid out as in
 * wva_workload_grid: each is [n_ticks * S], index t*S + s.
 *
 * Let c_0 be the fleet's (srv_cur_acc, srv_cur_replicas, srv_cur_cost), and f_t the fleet with srv_arrival_rpm,
 * srv_in_tokens and srv_out_tokens replaced by row t and its current-allocation columns replaced by c_t.
 *   - Candidate block t (records (t*S + s)*A + a) is byte for byte what wva_analyze returns for f_t: value =
 *     TransitionPenalty(c_t, .), and the keepAccelerator mask against c_t's accelerator (a masked pair is a nil
 *     record).
 *   - Winner block t (records t*S + s) is byte for byte wva_solve's winner block for f_t with unlimited = 1.
 *   - c_{t+1} is winner t's (acc, replicas, cost) when that winner is feasible, and c_t otherwise.  A zero-load
 *     winner with min_replicas 0 has accelerator WVA_ACC_NONE, 0 replicas and cost 0, and becomes exactly that.
 * This is the reference's Server.SetLoad(row t); Server.Calculate; SolveUnlimited; Server.ApplyDesiredAlloc per
 * tick, on a ServerSpec whose DesiredAlloc starts equal to its CurrentAlloc (the state ApplyDesiredAlloc leaves).
 * A spec built by the WVA adapters starts with an empty DesiredAlloc instead (internal/utils/utils.go:293).  The two
 * differ only for a server that has no winner at tick 0: the reference would then drop that server to the empty
 * allocation, while the controller (and this call) leaves it unchanged.
 *
 * Only unlimited mode is traced: limited mode's greedy pass couples the servers and runs on the host, and WVA always
 * runs unlimited (internal/utils/utils.go:170).  fleet->unlimited and the capacities are not read.  A trace can be
 * continued: the trace over ticks 0..L-1 equals the trace over 0..k-1 followed by the trace over k..L-1 on the fleet
 * whose srv_cur_* columns hold c_k.
 *
 * Sizing (DESIGN.md §3.13): CreateAllocation does not read the current allocation, so every tick's records are
 * sized in one batched pass with the workload grid's deduplication, and only the chain (mask, value, minimum,
 * advance) runs tick by tick, on the device.  A server is pinned when keepAccelerator is set, its current
 * accelerator is not WVA_ACC_NONE, and either that accelerator is WVA_ACC_UNKNOWN or min_replicas != 0: its
 * accelerator can never change, so only (s, srv_cur_acc[s]) is sized (nothing when unknown).  Every other server's
 * pairs are all sized, keepAccelerator ignored, since its current accelerator can change along the chain.
 *
 * The fleet becomes resident; wva_summarize returns WVA_ERR_STATE afterwards.  `candidates` (n_ticks*S*A entries)
 * may be NULL; `winners` has n_ticks*S entries.  n_ticks == 0 is valid (nothing is written).  WVA_ERR_BAD_ARG:
 * n_ticks < 0, a row list NULL with n_ticks * S > 0, or winners NULL.  WVA_ERR_UNSUPPORTED: S*A*n_ticks >= 2^31
 * (refused before the fleet is read), or the failures of wva_workload_grid for the pairs the call sizes: a load pair
 * outside the queue-size rule, a rescale loop that would not terminate, or too many stored-vector fallbacks.  This
 * set of refusals can be larger than the set of ticks at which wva_analyze(f_t) fails, but only through the pairs of
 * a server that is not pinned yet has keepAccelerator set, at ticks where the chain keeps them masked.  The call
 * never returns a result that differs from the per-tick composition.
 */
int wva_workload_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks, const float *arrival_rpm,
                       const int32_t *in_tokens, const int32_t *out_tokens, wva_allocs *candidates,
                       wva_allocs *winners);

/*
 * Rows of accelerator costs and model x accelerator performance data for wva_profile_grid.  Any pointer may be NULL:
 * that column is the fleet's own at every level.
 */
typedef struct wva_profile_rows {
    const float *acc_cost;                                            /* [L*A], index l*A + a                */
    const uint8_t *perf_present;                                      /* [L*M*A], index (l*M + m)*A + a      */
    const float *perf_alpha, *perf_beta, *perf_gamma, *perf_delta;    /* [L*M*A]                             */
    const int32_t *perf_acc_count, *perf_max_batch, *perf_at_tokens;  /* [L*M*A]                             */
} wva_profile_rows;

/*
 * Profile grid: Server.Calculate (as in wva_analyze) and SolveUnlimited's winner at each of n_levels caller-given
 * rows of accelerator costs and performance profiles, e.g. a price change, a spot price, an error in the fitted
 * alpha / beta / gamma / delta, or a new accelerator (listed with perf_present = 0, switched on per row).
 *
 * Let f_l be the fleet with acc_cost and the nine perf_* columns replaced by row l of `rows`.  Candidate block l
 * (records (l*S + s)*A + a) is byte for byte what wva_analyze returns for f_l, value = TransitionPenalty and the
 * keepAccelerator mask included.  Winner block l (records l*S + s) is wva_solve's winner block for f_l with
 * unlimited = 1: strict '<' from MaxFloat32, ties to the lower accelerator id.  acc_multiplicity, acc_type, the
 * capacities and fleet->unlimited are not read; every other column comes from `fleet`.  Each candidate block, with
 * its level's accelerator table, is a valid input for wva_solve_greedy, which serves limited mode.
 *
 * The current allocation's cost is srv_cur_cost as given, not re-priced at row l: in WVA it is the VariantCost
 * recorded in the variant's status, so block l is the decision at the first reconcile after the price change.
 *
 * Deduplication (DESIGN.md §3.14): CreateAllocation reads the accelerator's cost and AccCount only in the cost of
 * the allocation.  For a pair (s, a) the batch size at level l is N = srv_max_batch, or else
 * max(perf_max_batch * perf_at_tokens / out_tokens, 1) in 64 bits.  QueueAnalyzer.Size, rateStar, the replica count
 * and the final Analyze run once per distinct (s, a, bits of alpha, beta, gamma, delta, N) that some level uses as
 * a load pair; per level only the cost, the value and the minimum run.  A row list that changes only prices sizes
 * every pair once.
 *
 * The fleet becomes resident, as with every call that takes one; wva_summarize returns WVA_ERR_STATE afterwards.
 * `candidates` (n_levels*S*A entries) may be NULL; `winners` has n_levels*S entries.  n_levels == 0 is valid
 * (nothing is written).  `rows` NULL means every column is the fleet's own.  WVA_ERR_BAD_ARG: n_levels < 0, fleet
 * NULL or winners NULL.  WVA_ERR_UNSUPPORTED: S*A*n_levels >= 2^31 or n_levels*M*A >= 2^31 (refused before the
 * fleet is read), or exactly the levels on which wva_analyze of f_l fails the same way: a load pair outside the
 * queue-size rule (a level's perf_max_batch and perf_at_tokens can push N above 2^20), a rescale loop that would
 * not terminate, or too many stored-vector fallbacks.  Each key is sized only when some level uses it, so the
 * refusals are the union of the per-level ones.
 */
int wva_profile_grid(wva_handle *h, const wva_fleet *fleet, int32_t n_levels, const wva_profile_rows *rows,
                     wva_allocs *candidates, wva_allocs *winners);

/*
 * Profile trace: wva_workload_trace over ticks that also carry accelerator costs and performance profiles, e.g.
 * hourly spot or time-of-use prices, an accelerator brought online or withdrawn at some tick (perf_present), or a
 * serving-stack upgrade that lowers beta from some tick on.
 *
 * Let f_t be the fleet with srv_arrival_rpm, srv_in_tokens and srv_out_tokens replaced by row t of the three
 * workload lists ([L*S], index t*S + s; a NULL list is the fleet's own column at every tick), acc_cost and the nine
 * perf_* columns by row t of `rows` (wva_profile_rows' layout; a NULL column, or rows NULL, is the fleet's own), and
 * the current allocation (srv_cur_acc, srv_cur_replicas, srv_cur_cost) by c_t.
 *   - c_0 is the fleet's current allocation, not re-priced (in WVA it is the recorded VariantCost).
 *   - Candidate block t (records (t*S + s)*A + a) is byte for byte what wva_analyze returns for f_t, value =
 *     TransitionPenalty against c_t and the keepAccelerator mask against c_t included.
 *   - Winner block t (records t*S + s) is byte for byte wva_solve's winner block for f_t with unlimited = 1.
 *   - c_{t+1} is winner t's (acc, replicas, cost) when that winner is feasible, and c_t otherwise.  The cost carried
 *     forward is the winner's at tick t's prices (Server.ApplyDesiredAlloc), so the penalty at tick t+1 compares a
 *     cost recorded at the old prices with candidates priced at the new ones, as the controller does.
 * Only unlimited mode is traced; fleet->unlimited, the capacities, acc_type and acc_multiplicity are not read.  A
 * trace can be continued as wva_workload_trace's: the trace over ticks 0..L-1 equals the trace over 0..k-1 followed
 * by the trace over k..L-1 on the fleet whose srv_cur_* columns hold c_k.  With every profile column NULL the call
 * returns wva_workload_trace's result; with one tick it returns wva_profile_grid's for that row (on the fleet's own
 * load when the workload lists are NULL).
 *
 * Sizing (DESIGN.md §3.15): a load pair's record at tick t is fixed by (s, a, in_t, out_t, bits of alpha, beta,
 * gamma, delta and N at row t); the price and AccCount of row t enter only its cost.  Each distinct such key that some
 * tick uses as a load pair is sized once, in one batched pass, and only the chain runs tick by tick.  As in
 * wva_workload_trace, a pinned server sizes only its current pair and every other server sizes all its pairs,
 * keepAccelerator ignored.
 *
 * The fleet becomes resident; wva_summarize returns WVA_ERR_STATE afterwards.  `candidates` (n_ticks*S*A entries)
 * may be NULL; `winners` has n_ticks*S entries.  n_ticks == 0 is valid (nothing is written).  WVA_ERR_BAD_ARG:
 * n_ticks < 0, fleet NULL or winners NULL.  WVA_ERR_UNSUPPORTED: S*A*n_ticks >= 2^31 or n_ticks*M*A >= 2^31 (refused
 * before the fleet is read), or the union over ticks of wva_analyze(f_t)'s failures for the pairs the call sizes: a
 * load pair outside the queue-size rule (a tick's perf_max_batch, perf_at_tokens or out_tokens can push N above
 * 2^20), a rescale loop that would not terminate, or too many stored-vector fallbacks.  As with wva_workload_trace,
 * these can exceed the per-tick refusals only through the pairs of keep servers that are not pinned, and the result
 * never differs from the per-tick composition.  With a perf column the call also refuses when its distinct keys times
 * A reach 2^31 (at most S*A*n_ticks keys, so only with A*A*S*n_ticks >= 2^31); split the ticks over several calls
 * (continuation).
 */
int wva_profile_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks, const float *arrival_rpm,
                      const int32_t *in_tokens, const int32_t *out_tokens, const wva_profile_rows *rows,
                      wva_allocs *candidates, wva_allocs *winners);

/*
 * Load intervals: for each server, the exact float32 arrival rates in [rpm_lo[s], rpm_hi[s]] (req/min) at which
 * wva_load_grid's winner changes its decision, and the winner on each stretch in between.  An autoscaler can
 * skip a re-solve while the load stays inside the current interval, or publish the next scale-up and scale-down
 * rates.
 *
 * The decision key of a winner record is (feasible, acc, replicas, batch, cost, value, max_rate), compared
 * bitwise.  For server s the intervals partition [rpm_lo[s], rpm_hi[s]]: interval 0 starts at rpm_lo[s],
 * interval j covers [start_rpm[j], start_rpm[j+1]), and start_rpm[j] is the smallest float32 rate at which the
 * key differs from interval j-1's; adjacent stretches with the same key are one interval.  At every float32 rate
 * of an interval wva_load_grid's winner for s has the interval's key.  Record j (index s*M + j) is byte for byte
 * wva_load_grid's winner record for s at level start_rpm[j], latency columns (itl, ttft, rho) included; those vary
 * inside an interval and are reported at its start only.  A stretch without a feasible candidate is an interval
 * with a nil record.  Rate 0 is a point of its own (zeroLoadAllocation); the next interval starts at the smallest
 * positive float32 unless it has the same key.  With a TPS target or out_tokens 0 the decision does not read the
 * load, so such a server has one interval above rate 0.
 *
 * Above rate 0 each pair's key is a step function of the rate (DESIGN.md §3.10): the replica count never
 * decreases, and at a fixed count Analyze's rate check flips at most twice.  So each step is found exactly by a
 * bisection over float32 bit patterns, and the winner can change only where some pair steps.  The sizing runs once
 * per (server, accelerator), as in wva_load_grid.
 *
 * count[s] is the number of intervals written (1..M).  truncated[s] = 1 when the decision changes again in
 * (last start, rpm_hi[s]]: either M intervals were written first, or a pair of s would need more than INT32_MAX
 * replicas there (the int32 replicas column and the float-to-int conversion wrap, so the steps stop being
 * monotone).  In the second case the list stops at the last start below that rate, and count[s] = 0 when it is
 * rpm_lo[s] itself.  A truncated list's last interval ends at that next change, which is not reported.  Records
 * and start rates past count[s] are zero bytes.
 *
 * fleet->srv_arrival_rpm, fleet->unlimited and the capacities are not read.  The fleet becomes resident, and
 * wva_summarize returns WVA_ERR_STATE afterwards, as after wva_load_grid.  Columns of out->rec may be NULL (not
 * written).  WVA_ERR_BAD_ARG: out NULL, max_per_server < 1, rpm_lo, rpm_hi, count, truncated or start_rpm NULL
 * with S > 0, a bound that is NaN, infinite or negative, or rpm_lo[s] > rpm_hi[s].  WVA_ERR_UNSUPPORTED:
 * S * max_per_server >= 2^31; a server with rpm_hi[s] > 0 and a pair outside wva_analyze's queue-size rule (the
 * pair is a load pair at some rate of its range); or a range in which wva_load_grid fails: an interval start
 * whose solve fails the same way (a rescale loop that would not terminate, too many stored-vector fallbacks), or a
 * positive rate below
 * 60 * 2^-150 req/min on a server with a min_replicas-0 load pair.  There totalRate rounds to 0, the pair gets 0
 * replicas and Analyze solves at 0/0, whose rescale loop does not terminate in wva_load_grid (the Go reference
 * reports NaN latencies there).
 */
typedef struct wva_intervals {
    int32_t max_per_server; /* M: capacity per server                                            */
    int32_t *count;         /* [S] intervals written for server s                                */
    uint8_t *truncated;     /* [S] 1 if the decision changes again in (last start, rpm_hi[s]]    */
    float *start_rpm;       /* [S*M] first float32 arrival rate (req/min) of interval j           */
    wva_allocs rec;         /* [S*M] the per-server winner record at start_rpm                    */
} wva_intervals;

int wva_load_intervals(wva_handle *h, const wva_fleet *fleet, const float *rpm_lo, const float *rpm_hi,
                       wva_intervals *out);

/*
 * Solver.SolveGreedy + the best-effort saturation policies (pkg/solver/greedy.go:35-341) over a candidate
 * table the caller already holds: `candidates` (S*A, value = transition penalty as wva_analyze returns it) is
 * read, and modified where the reference scales best-effort allocations; `winners` (S) is written.  Host only
 * (no handle, no device work).  The multi-GPU limited mode shards candidate generation over the ranks,
 * all-gathers the candidate tables and calls this on every rank (SURVEY.md 8e): the greedy pass is one
 * sequential walk over a shared capacity map and does not shard.
 */
int wva_solve_greedy(const wva_fleet *fleet, wva_allocs *candidates, wva_allocs *winners);

/*
 * Latency sweep of QueueAnalyzer.Analyze over n_rates rates per (server, acc).  A point whose chain leaves
 * the streaming solve's exponent windows is re-run on the stored p[0..K] vector with the reference's rescale
 * loops, like a grid cell.  WVA_ERR_UNSUPPORTED when that rescale loop would not terminate (NaN rates), or when a
 * swept pair (every pair with a profile, in_tokens >= 0 and out_tokens >= 1, whatever its rate) is outside
 * wva_analyze's queue-size rule.
 */
int wva_sweep(wva_handle *h, const wva_fleet *fleet, int32_t n_rates, wva_sweep_out *out);

/*
 * What Manager.Optimize / Solver.Solve leave behind besides the per-server solution
 * (pkg/manager/manager.go:21-27): the per-accelerator-type totals of System.AllocateByType
 * (pkg/core/system.go:271-300) and the per-server orchestration differences of
 * CreateAllocationDiff (pkg/core/allocation.go:353-380, collected by pkg/solver/solver.go:51-58).
 * Any pointer may be NULL (that column is not written).
 *
 *   type_*  [T]: present = the type has an entry in the reference's allocationByType map (some
 *                server was allocated an accelerator of that type); count = sum of
 *                numReplicas * numInstances(model, acc) * multiplicity(acc); limit = capacity of the
 *                type (0 when the capacity map has no entry); cost = sum of the allocations' cost.
 *                The reference accumulates the float32 cost in Go map order (random); here the order
 *                is ascending server index.
 *   diff_*  [S]: old = CurrentAlloc of the server spec (always present: core/server.go:49), new = the
 *                solution's allocation, accelerator WVA_ACC_ABSENT / 0 replicas / cost 0 when the
 *                server got none ("none" in the reference); cost = newCost - oldCost.
 */
typedef struct wva_summary {
    uint8_t *type_present;
    int64_t *type_count;
    int32_t *type_limit;
    float *type_cost;
    int32_t *diff_old_acc;
    int32_t *diff_new_acc;
    int32_t *diff_old_replicas;
    int32_t *diff_new_replicas;
    float *diff_cost;
} wva_summary;

/* Summary of the most recent wva_solve / wva_resolve / wva_grid_solve / wva_size_grid on this handle (the winners
 * stay resident until the next call).  WVA_ERR_STATE when there is none, e.g. after wva_load_grid. */
int wva_summarize(wva_handle *h, wva_summary *out);

/* ---- MM1KModel (closed form) --------------------------------------------- */

/*
 * MM1KModel.Solve for n independent (K, lambda, mu) triples: pkg/analyzer/mm1kmodel.go:19-92 over
 * QueueModel.Solve (queuemodel.go:27-37).  The reference keeps this model next to the state-dependent one but
 * does not call it on the production path; it is here so that every model of pkg/analyzer has a device function.
 * One thread per triple, p[] is streamed (never stored).  math.Pow is restated from the Go standard library's
 * binary-powering algorithm (integer exponents only occur) so that host oracle and device agree bit for bit; it is
 * not pinned against the Go binary (no Go toolchain here), see DESIGN.md.
 * Columns have n entries (host pointers, any may be NULL); entries of an invalid triple are 0 except rho.
 * K < 0 is WVA_ERR_BAD_ARG (NewMM1KModel returns nil), K > 2^20 WVA_ERR_UNSUPPORTED.
 */
typedef struct wva_mm1k_out {
    uint8_t *is_valid;
    float *rho;
    float *avg_num_in_system;
    float *throughput;
    float *avg_resp_time;
    float *avg_serv_time;
    float *avg_wait_time;
    float *avg_queue_length;
    double *sum_p; /* sum of the state probabilities as the reference accumulates it */
} wva_mm1k_out;
int wva_mm1k_solve(wva_handle *h, int32_t n, const int32_t *K, const float *lambda, const float *mu,
                   wva_mm1k_out *out);

/* ---- streaming reconcile (BASELINE config 5) ---------------------------- */

/* Make `fleet` resident on the device (copies everything; caller memory is not
 * retained). Subsequent wva_update_load / wva_resolve calls reuse it. */
int wva_upload(wva_handle *h, const wva_fleet *fleet);
/* Replace the load columns of the resident fleet (any pointer may be NULL =
 * keep). Arrays have S entries. */
int wva_update_load(wva_handle *h, const float *arrival_rpm, const int32_t *in_tokens,
                    const int32_t *out_tokens);
/* wva_solve on the resident fleet. */
int wva_resolve(wva_handle *h, wva_allocs *candidates, wva_allocs *winners);

/* ---- device-resident variants (used by the multi-GPU driver and bench) --- */

/*
 * As wva_grid_solve / wva_resolve on the resident fleet, but `winners` columns are
 * DEVICE pointers (e.g. torch tensors) and nothing is copied to the host; the
 * work is enqueued on the handle's stream and the call returns without
 * synchronising.  wva_stream() exposes that cudaStream_t so that the caller can
 * order an NCCL all-gather of the winner records after it.
 */
int wva_grid_solve_device(wva_handle *h, const wva_grid *grid, wva_allocs *winners_dev);
int wva_resolve_device(wva_handle *h, wva_allocs *winners_dev);
void *wva_stream(wva_handle *h);
int wva_synchronize(wva_handle *h);

/* Number of kernel launches issued by this handle since creation. */
int64_t wva_launch_count(const wva_handle *h);
/* Device time (ms, CUDA events on the handle's stream) of the dominant kernel in
 * the most recent call, and of the whole call's device work. */
float wva_last_kernel_ms(const wva_handle *h);
float wva_last_device_ms(const wva_handle *h);

/* --- multi-GPU: all-gather of the per-rank winner block over peer memory --------------------
 * One process per GPU on one node.  Replaces the collective the reference does not have (its optimizer
 * is single-process; SURVEY.md 8e): each rank writes its block straight into every peer's gathered
 * buffer over NVLink and waits for the peers' blocks, in ONE kernel on the handle's stream.
 *   wva_xchg_create   allocate this rank's gathered buffer, return its 64-byte CUDA IPC handle
 *   wva_xchg_open     register the IPC handle of rank `peer_rank` (exchange the handles with any
 *                     host-side transport, e.g. torch.distributed all_gather_object); call for every rank
 *   wva_xchg_publish  enqueue the exchange of `src_block` (device memory, block_bytes); *gathered is the
 *                     device address of this step's [world][*slot_stride] byte buffer, valid once the
 *                     stream has passed the call (double-buffered by step parity)
 *   wva_xchg_error    after a synchronize: 1 if a peer never arrived (the kernel gives up after ~2 s)
 */
int wva_xchg_create(wva_handle *h, int world, int rank, size_t block_bytes, void *ipc_handle_out);
int wva_xchg_open(wva_handle *h, int peer_rank, const void *ipc_handle);
int wva_xchg_publish(wva_handle *h, const void *src_block, void **gathered, size_t *slot_stride);
int wva_xchg_error(wva_handle *h);
int wva_xchg_destroy(wva_handle *h);

#ifdef __cplusplus
}
#endif
#endif /* WVA_B200_H */

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
 * SLO trace: wva_workload_trace over ticks that also carry service-class targets, e.g. a time-of-day SLO schedule (a
 * premium class whose ITL is tightened during business hours and relaxed overnight), or a proposed target change
 * replayed over recorded traffic.  The controller re-reads the service classes on every reconcile, so a target edit
 * takes effect at the next tick, as a load change does.
 *
 * Let f_t be the fleet with srv_arrival_rpm, srv_in_tokens, srv_out_tokens, srv_slo_itl, srv_slo_ttft and srv_slo_tps
 * replaced by row t of the six lists (each [n_ticks * S], index t*S + s, in the units of the fleet's columns; a NULL
 * list is the fleet's own column at every tick) and its current allocation (srv_cur_acc, srv_cur_replicas,
 * srv_cur_cost) by c_t.
 *   - Candidate block t (records (t*S + s)*A + a) is byte for byte what wva_analyze returns for f_t, value =
 *     TransitionPenalty against c_t and the keepAccelerator mask against c_t included.
 *   - Winner block t (records t*S + s) is byte for byte wva_solve's winner block for f_t with unlimited = 1.
 *   - c_0 is the fleet's current allocation; c_{t+1} is winner t's (acc, replicas, cost) when that winner is
 *     feasible, and c_t otherwise (wva_workload_trace's rule).
 * Only unlimited mode is traced; fleet->unlimited and the capacities are not read.  A trace can be continued as
 * wva_workload_trace's: ticks 0..L-1 equal ticks 0..k-1 followed by ticks k..L-1 on the fleet whose srv_cur_* hold
 * c_k.  With the three target lists NULL the call returns wva_workload_trace's result on the same load rows; with one
 * tick it returns wva_slo_grid's for that row on the fleet whose load columns are the tick's.
 *
 * Sizing (DESIGN.md §3.17): Size, lambda* and rateStar read the tokens but not the rate, and each bisection reads only
 * its own target, so a search is fixed by (server, accelerator, in, out, which search, target bits).  Each distinct
 * search that some tick needs (its three targets not negative, the search's target > 0) runs once, in one batched
 * pass; per tick only lambda*, rateStar, the replica count and the final Analyze run, then the chain.  As in
 * wva_workload_trace, a pinned server sizes only its current pair and every other server sizes all its pairs,
 * keepAccelerator ignored.  With the fleet's own tokens, an ITL schedule of two values over 24 ticks runs three
 * searches per pair (one TTFT, two ITL) instead of 48.
 *
 * The fleet becomes resident; wva_summarize returns WVA_ERR_STATE afterwards.  `candidates` (n_ticks*S*A entries)
 * may be NULL; `winners` has n_ticks*S entries.  n_ticks == 0 is valid (nothing is written).  WVA_ERR_BAD_ARG:
 * n_ticks < 0, fleet NULL or winners NULL.  WVA_ERR_UNSUPPORTED: S*A*n_ticks >= 2^31 (refused before the fleet is
 * read); 2^31 or more search records (distinct search keys x A); or the union over ticks of wva_analyze(f_t)'s
 * failures for the pairs the call sizes: a load pair outside the queue-size rule, a rescale loop that would not
 * terminate (a NaN or tiny TPS target can cause one), or too many stored-vector fallbacks.  As with
 * wva_workload_trace, these can exceed the per-tick refusals only through the pairs of keep servers that are not
 * pinned, and the result never differs from the per-tick composition.  As in wva_slo_grid, a search that no tick's
 * reference would run (the ITL search after a failed TTFT search) does not fail the call.
 */
int wva_slo_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks, const float *arrival_rpm,
                  const int32_t *in_tokens, const int32_t *out_tokens, const float *slo_itl, const float *slo_ttft,
                  const float *slo_tps, wva_allocs *candidates, wva_allocs *winners);

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
 * Load margins: for each level l and server s, the exact stretch of float32 arrival rates around the level's rate
 * on which wva_load_grid's winner keeps its decision.  A controller can publish "scale down below lo_rpm, scale up
 * at hi_rpm" next to the desired replica count, or skip a re-solve while the load stays inside the stretch, and a
 * planner can see how far the real load may stray from each row of a forecast before the planned decision is wrong.
 *
 * Level l has wva_load_grid's semantics: the fleet with srv_arrival_rpm set to row l (index l*S + s; arrival_rpm
 * NULL is the fleet's own column at every level), against the fleet's own current allocation, solved in unlimited
 * mode.  The decision key is wva_load_intervals' (feasible, acc, replicas, batch, cost, value, max_rate), compared
 * bitwise.  Let r be row l's rate for s.  [lo_rpm, hi_rpm) is the maximal stretch of float32 rates in
 * [rpm_lo, rpm_hi] (entry l*S + s of each) that contains r and on which the key equals the key at r.  It is exactly
 * the interval that wva_load_intervals over the same window, with max_per_server large enough, reports as containing
 * r, and hi_rpm is the start of the next interval in that list.  Rate 0 is a point of its own, as there.
 *
 * at, below and above are byte for byte wva_load_grid's winner records at r, at nextafterf(lo_rpm, 0) and at
 * hi_rpm, latency columns included (taken at those exact rates).  Flags:
 *   WVA_MARGIN_LO_OPEN    no change in [rpm_lo, r]: lo_rpm = rpm_lo, `below` is zero bytes;
 *   WVA_MARGIN_HI_OPEN    no change in (r, rpm_hi]: hi_rpm = +Inf, `above` is zero bytes;
 *   WVA_MARGIN_TRUNCATED  a pair of s would need more than INT32_MAX replicas (where the steps stop being monotone,
 *                         see wva_load_intervals) at hi_rpm, which is then the first such rate above r, or at r
 *                         itself, where lo_rpm = hi_rpm = r and `below` is zero bytes.  `above` is zero bytes.
 *
 * Each pair's state is a step function of the rate (DESIGN.md §3.10), so the call walks from r up to the first
 * change of the winner's key and down to the last one, each step found by a bisection over float32 bit patterns
 * (§3.19).  The sizing runs once per (server, accelerator), as in wva_load_grid.
 *
 * fleet->unlimited and the capacities are not read; fleet->srv_arrival_rpm only when arrival_rpm is NULL.  The
 * fleet becomes resident, and wva_summarize returns WVA_ERR_STATE afterwards.  Columns of at, below and above may be
 * NULL (not written).  n_levels == 0 is valid (nothing is written).  WVA_ERR_BAD_ARG: n_levels < 0, out NULL,
 * rpm_lo, rpm_hi, lo_rpm, hi_rpm or flags NULL with S*n_levels > 0, a rate, rpm_lo or rpm_hi that is NaN, infinite
 * or negative, or rpm_lo > r or r > rpm_hi.  WVA_ERR_UNSUPPORTED: 3*S*n_levels >= 2^31 (three records per level and
 * server; refused before the fleet is read), or where wva_load_intervals refuses, for the servers with some level whose rpm_hi > 0: a pair outside
 * wva_analyze's queue-size rule, a solve at r, below lo_rpm or at hi_rpm whose rescale loop would not terminate, too
 * many stored-vector fallbacks, or a window holding a positive rate below 60 * 2^-150 req/min on a server with a
 * min_replicas-0 load pair.
 */
#define WVA_MARGIN_LO_OPEN 1
#define WVA_MARGIN_HI_OPEN 2
#define WVA_MARGIN_TRUNCATED 4

typedef struct wva_margins {
    float *lo_rpm;    /* [L*S] first float32 rate of the stretch that holds the level's rate                   */
    float *hi_rpm;    /* [L*S] first float32 rate above it at which the decision key differs (+Inf: none)    */
    uint8_t *flags;   /* [L*S] WVA_MARGIN_*                                                                   */
    wva_allocs at;    /* [L*S] wva_load_grid's winner record at the level's rate                              */
    wva_allocs below; /* [L*S] wva_load_grid's winner record at the largest float32 below lo_rpm              */
    wva_allocs above; /* [L*S] wva_load_grid's winner record at hi_rpm                                        */
} wva_margins;

int wva_load_margins(wva_handle *h, const wva_fleet *fleet, int32_t n_levels,
                     const float *arrival_rpm /* [L*S], NULL: the fleet's own column at every level */,
                     const float *rpm_lo, const float *rpm_hi /* [L*S] search window, req/min */, wva_margins *out);

/*
 * Load margin trace: wva_load_margins along a replayed reconcile.  Every level of wva_load_margins is solved against
 * the fleet's own current allocation c_0, but a controller that follows a forecast holds, at tick t, the current
 * allocation c_t that wva_workload_trace carries into tick t: the last feasible winner of ticks 0..t-1, or c_0 when
 * there is none.  TransitionPenalty and keepAccelerator read it, so the margins around tick t's load depend on the
 * chain.  This call gives them in one call, without one upload and one sizing per tick.
 *
 * Rows are laid out as in wva_load_margins (index t*S + s, n_ticks*S entries per column of out), over load only:
 * the tokens are the fleet's own columns.  Let f_t be the fleet with srv_arrival_rpm = row t of arrival_rpm and
 * its current-allocation columns (srv_cur_acc, srv_cur_replicas, srv_cur_cost) = c_t, where c_{t+1} is winner t's
 * (acc, replicas, cost) when that winner is feasible and c_t otherwise.  A zero-load winner with min_replicas 0 has
 * accelerator WVA_ACC_NONE, 0 replicas and cost 0, and becomes exactly that.
 *   - Block t of lo_rpm, hi_rpm, flags, at, below and above is byte for byte wva_load_margins(f_t) with one level:
 *     rate row t, window row t (rpm_lo, rpm_hi).  The load moves at tick t only; the ticks before t do not read it,
 *     so c_t does not move with it.
 *   - Together, the `at` blocks are byte for byte wva_workload_trace's winners on the same rate rows with token rows
 *     equal to the fleet's own columns.  That is a check of the chain that needs no oracle.
 * A trace can be continued as wva_workload_trace's can: ticks 0..L-1 equal ticks 0..k-1 followed by ticks k..L-1 on
 * the fleet whose srv_cur_* columns hold c_k (Fleet.apply_winners over the `at` blocks in Python).
 *
 * Sizing (DESIGN.md §3.21): phase 1 is wva_load_margins', with keepAccelerator honoured on the pinned servers only
 * (wva_workload_trace's rule: keepAccelerator set, a current accelerator other than WVA_ACC_NONE, and either
 * WVA_ACC_UNKNOWN or min_replicas != 0), since any other server's current accelerator can change along the chain.
 * One kernel then walks each server's ticks for c_t, and the margin walk and the records read c_t.
 *
 * Only unlimited mode is covered; fleet->unlimited and the capacities are not read.  The fleet becomes resident,
 * and wva_summarize returns WVA_ERR_STATE afterwards.  Columns of at, below and above may be NULL (not written).
 * n_ticks == 0 and S == 0 are valid (nothing is written).  WVA_ERR_BAD_ARG: n_ticks < 0, out NULL, arrival_rpm,
 * rpm_lo, rpm_hi, lo_rpm, hi_rpm or flags NULL with S*n_ticks > 0, or a row that wva_load_margins(f_t) refuses
 * (NaN, infinite or negative, or the rate outside its window).  WVA_ERR_UNSUPPORTED: 3*S*n_ticks >= 2^31 (refused
 * before the fleet is read), or where wva_load_margins(f_t) refuses at some tick t.  This set of refusals can be
 * larger than the union over t of what wva_load_margins(f_t) refuses, but only through the pairs of a server that
 * is not pinned yet has keepAccelerator set, at ticks where the chain keeps them masked.  The call never returns a
 * result that differs from the per-tick composition.
 */
int wva_load_margin_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks,
                          const float *arrival_rpm /* [L*S], required */,
                          const float *rpm_lo, const float *rpm_hi /* [L*S] windows, req/min */, wva_margins *out);

/*
 * Workload margins: wva_load_margins and wva_load_margin_trace at rows that carry their own token lengths, as the
 * collector reports them on every tick (arrival rate, AvgInTokens, AvgOutTokens).  A reconcile loop can skip its
 * re-solve while the load stays inside a row's stretch and the tokens stay the row's, and a planner sees how far the
 * load of each row of a (rate, in, out) forecast may stray.  Without this call that takes one wva_load_margins per
 * row, each re-uploading and re-sizing the fleet with its token columns rewritten.
 *
 * Rows are laid out as in wva_workload_grid: arrival_rpm, in_tokens, out_tokens, rpm_lo and rpm_hi are [L*S], index
 * l*S + s, with L = n_levels or n_ticks, and so is every column of out.  arrival_rpm is required; a NULL token list
 * is the fleet's own column at every row.
 *   - Grid, level l.  Let f_l be the fleet with srv_arrival_rpm, srv_in_tokens and srv_out_tokens replaced by row
 *     l.  Block l of lo_rpm, hi_rpm, flags, at, below and above is byte for byte wva_load_margins(f_l) with one
 *     level: rate row l, window row l.  Together, the `at` blocks are wva_workload_grid's winners on the same rows.
 *   - Trace, tick t.  Let f_t be that fleet with row t and srv_cur_* = c_t, the allocation wva_workload_trace
 *     carries into tick t on the same (rate, in, out) rows.  Block t is byte for byte wva_load_margins(f_t) with one
 *     level, and the `at` blocks are wva_workload_trace's winners.  A trace continues as wva_workload_trace's does:
 *     ticks 0..L-1 equal ticks 0..k-1 followed by ticks k..L-1 on the fleet whose srv_cur_* hold c_k
 *     (Fleet.apply_winners over the `at` blocks in Python).
 *   - With both token lists NULL the result is byte for byte wva_load_margins (grid) or wva_load_margin_trace
 *     (trace) on the same rate rows and windows.
 * A new rate inside [lo_rpm, hi_rpm) keeps the row's decision when the new tokens equal the row's; the stretch says
 * nothing about other tokens.
 *
 * Sizing (DESIGN.md §3.22): QueueAnalyzer.Size, lambda* and rateStar read the tokens but not the rate, so phase 1
 * runs once per distinct (server, accelerator, in_tokens, out_tokens) over the rows whose window top rpm_hi is above
 * 0 and whose tokens class a pair as a load (in_tokens >= 0, out_tokens >= 1); on a trace with keepAccelerator
 * honoured on the pinned servers only, as wva_workload_trace does.  The walk then reads each row's tokens.
 *
 * Only unlimited mode is covered; fleet->unlimited and the capacities are not read, nor are srv_arrival_rpm and, where
 * a token list is given, its column.  The fleet becomes resident, and wva_summarize returns WVA_ERR_STATE afterwards.
 * Columns of at, below and above may be NULL (not written).  L == 0 and S == 0 are valid (nothing is written).
 * WVA_ERR_BAD_ARG: L < 0, out NULL, arrival_rpm, rpm_lo, rpm_hi, lo_rpm, hi_rpm or flags NULL with S*L > 0, or a row
 * that wva_load_margins refuses (NaN, infinite or negative, or the rate outside its window).  WVA_ERR_UNSUPPORTED:
 * 3*S*L >= 2^31 (refused before the fleet is read); distinct keys x A >= 2^31; or, for the grid, exactly where
 * wva_load_margins(f_l) refuses at some level l: a pair outside the queue-size rule at row l's out_tokens, a rescale
 * loop that would not terminate, too many stored-vector fallbacks, or a window holding a positive rate below
 * 60 * 2^-150 req/min on a server with a min_replicas-0 load pair.  A token pair used only at rows whose window is
 * [0, 0] is never sized and does not fail the call.  The trace's refusals can be larger than the union over t of what
 * wva_load_margins(f_t) refuses, but only through the pairs of a server that is not pinned yet has keepAccelerator
 * set, at ticks where the chain keeps them masked.  The call never returns a result that differs from the per-row
 * composition.
 */
int wva_workload_margins(wva_handle *h, const wva_fleet *fleet, int32_t n_levels, const float *arrival_rpm,
                         const int32_t *in_tokens, const int32_t *out_tokens,
                         const float *rpm_lo, const float *rpm_hi, wva_margins *out);
int wva_workload_margin_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks, const float *arrival_rpm,
                              const int32_t *in_tokens, const int32_t *out_tokens,
                              const float *rpm_lo, const float *rpm_hi, wva_margins *out);

/*
 * Profile margins: wva_workload_margins and wva_workload_margin_trace at rows that also carry their own accelerator
 * costs and performance profiles, as wva_profile_grid and wva_profile_trace take them: hourly spot or time-of-use
 * prices, an accelerator brought online or withdrawn, a beta change.  A planner replaying a day of prices sees how
 * far the load of each row may stray at that row's prices.  Without this call that takes one wva_load_margins per
 * row, each re-uploading and re-sizing the fleet with its acc_cost and perf_* columns rewritten.
 *
 * Rows: arrival_rpm, in_tokens, out_tokens, rpm_lo and rpm_hi are [L*S], index l*S + s, with L = n_levels or n_ticks;
 * `rows` has wva_profile_rows' layout (acc_cost [L*A], each perf_* [L*M*A]); every column of out is [L*S].
 * arrival_rpm is required; a NULL token list, a NULL profile column, or rows NULL, is the fleet's own column at every
 * row.
 *   - Grid, level l.  Let f_l be the fleet with srv_arrival_rpm, srv_in_tokens, srv_out_tokens, acc_cost and the
 *     nine perf_* columns replaced by row l.  Block l of lo_rpm, hi_rpm, flags, at, below and above is byte for byte
 *     wva_load_margins(f_l) with one level: rate row l, window row l.  The `at` blocks are wva_profile_trace's winner
 *     for each row alone (one tick on f_l); with arrival_rpm the fleet's own column at every row and NULL token lists
 *     they are wva_profile_grid's winners.
 *   - Trace, tick t.  Let f_t be that fleet with row t and srv_cur_* = c_t, the allocation wva_profile_trace carries
 *     into tick t on the same rows: the cost it carries is the winner's at its own tick's prices, and c_0's
 *     srv_cur_cost is not re-priced.  Block t is byte for byte wva_load_margins(f_t) with one level, and the `at`
 *     blocks are wva_profile_trace's winners.  The trace continues as wva_profile_trace's does: ticks 0..L-1 equal
 *     ticks 0..k-1 followed by ticks k..L-1 on the fleet whose srv_cur_* hold c_k.
 *   - With every profile column NULL the result is byte for byte wva_workload_margins (grid) or
 *     wva_workload_margin_trace (trace) on the same load rows and windows.
 * A new rate inside [lo_rpm, hi_rpm) keeps the row's decision when the tokens, prices and profiles stay the row's.
 *
 * Sizing (DESIGN.md §3.23): price and AccCount enter only the cost, price x NumInstances x replicas, and alpha .. delta
 * and N fix a pair's sizing without reading the rate.  So a pair's phase-1 record at row l is fixed by its key (s, a,
 * in_l, out_l, bits of alpha, beta, gamma, delta at row l, N at row l), N being srv_max_batch or else
 * max(perf_max_batch * perf_at_tokens / out_tokens, 1) in 64 bits.  Each distinct key is sized once over the rows
 * whose window top rpm_hi is above 0 and at which the pair is a load pair (perf_present at the row, in_tokens >= 0,
 * out_tokens >= 1); on a trace keepAccelerator is honoured on the pinned servers only.  Without a perf column the keys
 * are wva_workload_margins' (server, in, out) rows, and the call sizes the same pairs in the same order.
 *
 * Only unlimited mode is covered; fleet->unlimited, the capacities, acc_type and acc_multiplicity are not read, nor
 * are srv_arrival_rpm and the columns whose row lists are given.  The fleet becomes resident, and wva_summarize
 * returns WVA_ERR_STATE afterwards.  Columns of at, below and above may be NULL (not written).  L == 0 and S == 0 are
 * valid (nothing is written).  WVA_ERR_BAD_ARG: L < 0, out NULL, arrival_rpm, rpm_lo, rpm_hi, lo_rpm, hi_rpm or flags
 * NULL with S*L > 0, or a row that wva_load_margins refuses.  WVA_ERR_UNSUPPORTED: 3*S*L >= 2^31 or L*M*A >= 2^31
 * (both refused before the fleet is read); distinct key pairs x A >= 2^31; or, for the grid, exactly where
 * wva_load_margins(f_l) refuses at some level l (a row's perf_max_batch, perf_at_tokens or out_tokens can push N
 * above 2^20).  A key used only at rows whose window is [0, 0] is never sized and does not fail the call.  The trace's
 * refusals can be larger than the union over t of what wva_load_margins(f_t) refuses, but only through the pairs of a
 * server that is not pinned yet has keepAccelerator set.  The call never returns a result that differs from the
 * per-row composition.
 */
int wva_profile_margins(wva_handle *h, const wva_fleet *fleet, int32_t n_levels, const float *arrival_rpm,
                        const int32_t *in_tokens, const int32_t *out_tokens, const wva_profile_rows *rows,
                        const float *rpm_lo, const float *rpm_hi, wva_margins *out);
int wva_profile_margin_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks, const float *arrival_rpm,
                             const int32_t *in_tokens, const int32_t *out_tokens, const wva_profile_rows *rows,
                             const float *rpm_lo, const float *rpm_hi, wva_margins *out);

/*
 * SLO margins: wva_workload_margins and wva_workload_margin_trace at rows that also carry their own ITL, TTFT and
 * TPS targets, as wva_slo_trace takes them: a premium class whose ITL is tightened during business hours, or a
 * proposed target change replayed over recorded traffic.  A planner sees how far the load of each row may stray at
 * that row's targets.  Without this call that takes one wva_load_margins per row, each re-uploading and re-sizing the
 * fleet with its srv_slo_* columns rewritten.
 *
 * Rows: arrival_rpm, in_tokens, out_tokens, slo_itl, slo_ttft, slo_tps, rpm_lo and rpm_hi are [L*S], index l*S + s,
 * with L = n_levels or n_ticks, as in wva_slo_trace; every column of out is [L*S].  arrival_rpm is required; a NULL
 * token or target list is the fleet's own column at every row.
 *   - Grid, level l.  Let f_l be the fleet with srv_arrival_rpm, srv_in_tokens, srv_out_tokens, srv_slo_itl,
 *     srv_slo_ttft and srv_slo_tps replaced by row l.  Block l of lo_rpm, hi_rpm, flags, at, below and above is byte
 *     for byte wva_load_margins(f_l) with one level: rate row l, window row l.  The `at` blocks are wva_slo_trace's
 *     winner for each row alone (one tick on f_l); with arrival_rpm the fleet's own column at every row and NULL
 *     token lists they are wva_slo_grid's winners.
 *   - Trace, tick t.  Let f_t be that fleet with row t and srv_cur_* = c_t, the allocation wva_slo_trace carries into
 *     tick t on the same rows.  Block t is byte for byte wva_load_margins(f_t) with one level, and the `at` blocks
 *     are wva_slo_trace's winners.  The trace continues as wva_slo_trace's does: ticks 0..L-1 equal ticks 0..k-1
 *     followed by ticks k..L-1 on the fleet whose srv_cur_* hold c_k.
 *   - With all three target lists NULL the result is byte for byte wva_workload_margins (grid) or
 *     wva_workload_margin_trace (trace) on the same load rows and windows, with the same launch count.
 * A new rate inside [lo_rpm, hi_rpm) keeps the row's decision when the tokens and targets stay the row's.
 *
 * Sizing (DESIGN.md §3.24): QueueAnalyzer.Size reads the ITL and TTFT targets and whether the TPS target is positive,
 * and the tail's totalRate reads the TPS target; none of them reads the rate.  So a pair's phase-1 record at row l is
 * fixed by (s, a, in_l, out_l, bits of ITL_l, TTFT_l and TPS_l), and each distinct key is sized once over the rows
 * whose window top rpm_hi is above 0 and whose tokens class a pair as a load (in_tokens >= 0, out_tokens >= 1); on a
 * trace with keepAccelerator honoured on the pinned servers only.  With NULL target lists the keys are
 * wva_workload_margins' (server, in, out) rows, and the call sizes the same pairs in the same order.  A key with a
 * negative target is sized like any other (Size makes its pairs nil), as wva_load_margins(f_l) sizes it.
 *
 * Only unlimited mode is covered; fleet->unlimited and the capacities are not read, nor are srv_arrival_rpm and the
 * columns whose row lists are given.  srv_has_target still gates a server's pairs.  The fleet becomes resident, and
 * wva_summarize returns WVA_ERR_STATE afterwards.  Columns of at, below and above may be NULL (not written).  L == 0
 * and S == 0 are valid (nothing is written).  WVA_ERR_BAD_ARG: L < 0, out NULL, arrival_rpm, rpm_lo, rpm_hi, lo_rpm,
 * hi_rpm or flags NULL with S*L > 0, or a row that wva_load_margins refuses.  WVA_ERR_UNSUPPORTED: 3*S*L >= 2^31
 * (refused before the fleet is read); distinct key pairs x A >= 2^31; or, for the grid, exactly where
 * wva_load_margins(f_l) refuses at some level l, a NaN or tiny TPS target under a window top above 0 among them.  A
 * key used only at rows whose window is [0, 0] is never sized and does not fail the call.  The trace's refusals can
 * be larger than the union over t of what wva_load_margins(f_t) refuses, but only through the pairs of a server that
 * is not pinned yet has keepAccelerator set.  The call never returns a result that differs from the per-row
 * composition.
 */
int wva_slo_margins(wva_handle *h, const wva_fleet *fleet, int32_t n_levels, const float *arrival_rpm,
                    const int32_t *in_tokens, const int32_t *out_tokens,
                    const float *slo_itl, const float *slo_ttft, const float *slo_tps,
                    const float *rpm_lo, const float *rpm_hi, wva_margins *out);
int wva_slo_margin_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks, const float *arrival_rpm,
                         const int32_t *in_tokens, const int32_t *out_tokens,
                         const float *slo_itl, const float *slo_ttft, const float *slo_tps,
                         const float *rpm_lo, const float *rpm_hi, wva_margins *out);

/*
 * Price thresholds: for each server s and accelerator a, the exact accelerator price at which s's unlimited
 * winner leaves a.  Let f(p) be the fleet with acc_cost[a] = p, solved in unlimited mode.
 *
 * threshold[s*A + a] is the smallest float32 p in [+0, MaxFloat32] at which s's wva_solve winner on f(p) is not
 * a's candidate, and +Inf when a's candidate wins at every such p.  a's candidate wins at every price below the
 * threshold (DESIGN.md §3.16): CreateAllocation reads p only in the cost of a's own candidates (cost = p *
 * NumInstances * replicas), the current cost srv_cur_cost is not re-priced (as in wva_profile_grid), and
 * TransitionPenalty of a's candidate never decreases as p grows.  So 0 means a never wins at a non-negative
 * price: a nil or keepAccelerator-masked pair, a NaN value, or a candidate beaten at cost 0.  A candidate whose
 * value does not read p (same accelerator and replica count as the current allocation, penalty 0) gets 0 or
 * +Inf.  Negative prices are outside the contract.  Column a of threshold does not depend on the fleet's own
 * acc_cost[a].
 *
 * above[s*A + a] is byte for byte wva_profile_grid's winner record for s at the row acc_cost[a] = threshold:
 * where s goes once a is too expensive (a nil record when no other candidate can win).  It is zero bytes where
 * the threshold is +Inf.  candidates (S*A) is byte for byte what wva_analyze returns for the fleet.  above and
 * candidates may be NULL, and so may any of their columns (not written).
 *
 * Only unlimited mode is covered: fleet->unlimited and the capacities are not read.  The fleet becomes
 * resident, and wva_summarize returns WVA_ERR_STATE afterwards.  WVA_ERR_BAD_ARG: threshold NULL with S*A > 0.
 * WVA_ERR_UNSUPPORTED: whatever wva_analyze refuses (the queue-size rule, a rescale loop that would not
 * terminate, too many stored-vector fallbacks), and, before any kernel is launched, the inputs on which a
 * candidate's value could decrease as its price grows: a penalty factor (tun.accel_penalty_factor) that is NaN,
 * negative or infinite, or an srv_cur_cost that is NaN or infinite on a server with a pair wva_analyze does not
 * class nil (a pair it sizes, or a zero-load candidate).
 */
int wva_price_thresholds(wva_handle *h, const wva_fleet *fleet, float *threshold /* [S*A] */,
                         wva_allocs *above /* [S*A], may be NULL */, wva_allocs *candidates /* [S*A], may be NULL */);

/*
 * Price threshold grid and trace: wva_price_thresholds at every row of a forecast, e.g. how many units of
 * accelerator a the fleet uses at each price of a in each hour.  The rows are laid out as in wva_workload_grid:
 * arrival_rpm, in_tokens and out_tokens are [L*S], index l*S + s, with L = n_levels or n_ticks.  arrival_rpm is
 * required; a NULL token list is the fleet's own column at every row.  Output block l of threshold, above and
 * candidates is records (l*S + s)*A + a; of winners, l*S + s.
 *
 *   - Grid, level l.  Let f_l be the fleet with row l of the three lists.  Block l of threshold, above and
 *     candidates is byte for byte what wva_price_thresholds(f_l) returns, and winner block l is wva_workload_grid's.
 *   - Trace, tick t.  Let f_t be the fleet with row t and current allocation c_t, the current allocation
 *     wva_workload_trace carries into tick t (the last feasible winner of ticks 0..t-1, the fleet's own without
 *     one).  Block t is byte for byte wva_price_thresholds(f_t), and winners are wva_workload_trace's.  So the price
 *     of a changes at tick t only: the ticks before t do not read it, c_t does not move, and the argument of
 *     wva_price_thresholds applies to f_t as it stands.  A price that changes at every tick is not offered: through
 *     the chain a's winning at tick t-1 changes c_t, and nothing shows its winning prices are then one interval
 *     (DESIGN.md §3.20).
 *
 * Only unlimited mode is covered: fleet->unlimited and the capacities are not read.  The fleet becomes resident,
 * and wva_summarize returns WVA_ERR_STATE afterwards.  above and candidates may be NULL, and so may any of their
 * columns (not written); winners may not.  L == 0 is valid (nothing is written).  WVA_ERR_BAD_ARG: L < 0, winners
 * NULL, arrival_rpm NULL with L*S > 0, threshold NULL with L*S*A > 0.  WVA_ERR_UNSUPPORTED, with wva_last_error
 * naming the rule and, for a current cost, the server and the level or tick:
 *   - whatever wva_workload_grid (grid) or wva_workload_trace (trace) refuses on the same rows, and L*S*A >= 2^31;
 *   - before any launch, a penalty factor that is NaN, negative or infinite;
 *   - grid, before any launch: an srv_cur_cost that is NaN or infinite on a server with a pair that wva_analyze(f_l)
 *     does not class nil at some level l;
 *   - trace, after the winners are known: a c_t cost that is NaN or infinite on a server with a pair that
 *     wva_analyze(f_t) does not class nil.  A carried cost can be +Inf: a winner with c_t's accelerator and replica
 *     count has value 0 whatever its cost, and an acc_cost near MaxFloat32 makes that cost overflow.  The outputs
 *     are then unspecified.
 * Each is a case in which wva_price_thresholds refuses some level's or tick's fleet.
 */
int wva_price_threshold_grid(wva_handle *h, const wva_fleet *fleet, int32_t n_levels, const float *arrival_rpm,
                             const int32_t *in_tokens, const int32_t *out_tokens, float *threshold /* [L*S*A] */,
                             wva_allocs *above /* [L*S*A], may be NULL */,
                             wva_allocs *candidates /* [L*S*A], may be NULL */, wva_allocs *winners /* [L*S] */);
int wva_price_threshold_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks, const float *arrival_rpm,
                              const int32_t *in_tokens, const int32_t *out_tokens, float *threshold /* [L*S*A] */,
                              wva_allocs *above /* [L*S*A], may be NULL */,
                              wva_allocs *candidates /* [L*S*A], may be NULL */, wva_allocs *winners /* [L*S] */);

/*
 * Profile price thresholds: the price threshold grid and trace at rows that also carry their own accelerator costs
 * and performance profiles, e.g. a day of hourly prices on every accelerator, an AccCount or beta change after an
 * upgrade, or an accelerator that comes online at some hour.  The load rows are laid out as in
 * wva_price_threshold_grid, the profile rows as in wva_profile_trace (acc_cost [L*A], each perf_* [L*M*A]).
 * arrival_rpm is required; a NULL token list, a NULL profile column or rows == NULL is the fleet's own column at every
 * row.  The output layout is wva_price_threshold_grid's.
 *
 *   - Grid, level l.  Let f_l be the fleet with row l of the three load lists, of acc_cost and of the nine perf_*
 *     columns.  Block l of threshold, above and candidates is byte for byte what wva_price_thresholds(f_l) returns,
 *     and winner block l is wva_solve(f_l)'s with unlimited = 1.  With arrival_rpm the fleet's own column at every
 *     row and NULL token lists, candidates and winners are wva_profile_grid's.
 *   - Trace, tick t.  Let f_t be that fleet with srv_cur_* = c_t, the allocation wva_profile_trace carries into tick
 *     t, whose cost is at its own tick's prices.  Block t is byte for byte wva_price_thresholds(f_t), and candidates
 *     and winners are wva_profile_trace's.  The trace continues as wva_profile_trace's does: ticks 0..L-1 equal
 *     ticks 0..k-1 of one call followed by ticks k..L-1 of a call on the fleet with c_k in its srv_cur_* columns.
 *
 * Column a of threshold and of above, in block l, does not read row l's acc_cost[a]: a's price moves at row l
 * alone, and every other record of the row keeps the row's prices.  srv_cur_cost is not re-priced.  With every
 * profile column NULL the result is byte for byte wva_price_threshold_grid's or wva_price_threshold_trace's on the
 * same load rows, with the same kernel launches.
 *
 * Only unlimited mode is covered.  The fleet becomes resident, and wva_summarize returns WVA_ERR_STATE afterwards.
 * above and candidates may be NULL, and so may any of their columns; winners may not.  L == 0 is valid.
 * WVA_ERR_BAD_ARG: L < 0, winners NULL, arrival_rpm NULL with L*S > 0, threshold NULL with L*S*A > 0.
 * WVA_ERR_UNSUPPORTED, with wva_last_error naming the rule and, for a current cost, the server and the level or tick:
 *   - whatever wva_profile_trace (trace) or its grid mode (grid) refuses on the same rows: L*S*A >= 2^31,
 *     L*M*A >= 2^31, 2^31 or more key pairs x accelerators, and the sizing's own refusals;
 *   - wva_price_threshold_grid's and _trace's price rules, at f_l or f_t: a penalty factor that is NaN, negative or
 *     infinite, and a current cost that is NaN or infinite on a server with a pair not classed nil at that row,
 *     under the row's perf_present, rate and tokens.  The grid checks before any launch, the trace after the
 *     winners are known.  A carried cost can be +Inf or NaN at a row with an infinite or NaN price: a winner with
 *     c_t's accelerator and replica count has value 0 whatever its cost.
 */
int wva_profile_price_threshold_grid(wva_handle *h, const wva_fleet *fleet, int32_t n_levels,
                                     const float *arrival_rpm, const int32_t *in_tokens, const int32_t *out_tokens,
                                     const wva_profile_rows *rows, float *threshold /* [L*S*A] */,
                                     wva_allocs *above /* [L*S*A], may be NULL */,
                                     wva_allocs *candidates /* [L*S*A], may be NULL */,
                                     wva_allocs *winners /* [L*S] */);
int wva_profile_price_threshold_trace(wva_handle *h, const wva_fleet *fleet, int32_t n_ticks,
                                      const float *arrival_rpm, const int32_t *in_tokens, const int32_t *out_tokens,
                                      const wva_profile_rows *rows, float *threshold /* [L*S*A] */,
                                      wva_allocs *above /* [L*S*A], may be NULL */,
                                      wva_allocs *candidates /* [L*S*A], may be NULL */,
                                      wva_allocs *winners /* [L*S] */);

/*
 * SLO bounds: for each (server s, accelerator a) and search w (0: TTFT, 1: ITL), the exact targets at which the
 * reference's candidate turns nil and at which its target stops binding.  Entry (s*A + a)*2 + w of each column.
 *
 * BinarySearch (utils.go:26-70) decides from the target t > 0 and two values that do not depend on it, y_lo =
 * eval(lambda_min) and y_hi = eval(lambda_max) (EvalTTFT or EvalITL, both from one Model.Solve at that lambda in
 * req/ms), which class t falls in:
 *   NIL       "target is below the bounded region": Size fails and the candidate is nil;
 *   FREE      lambda* = lambda_max exactly (within tolerance of y_hi, or above the bounded region);
 *   SEARCHED  within tolerance of y_lo, or the bisection runs.
 * Over the positive float32 targets up to +Inf the classes come in one order (DESIGN.md §3.18): rising (y_lo <
 * y_hi) NIL, SEARCHED, FREE; otherwise FREE, SEARCHED, NIL.  Any stretch may be empty.  b1 <= b2 split them: t is
 * in the first stretch when !(t >= b1), in the last when t >= b2, else in the middle one.  b1 or b2 is NaN where
 * the stretches before it reach through +Inf (no positive target is past it).  Two consequences are exact:
 *   - t in the NIL stretch of w: the candidate is nil whatever the other targets are;
 *   - t in the FREE stretch of w: the candidate is byte for byte the one with w's target 0 and the other targets
 *     unchanged (lambda* is lambda_max, bit for bit, in both).
 * So a server whose candidates are all NIL at t has a nil winner, and one whose candidates that read the target
 * are all FREE at t has its winner at target 0.
 *
 * kind: 0 target not read (a pair that is not a load pair, or a model of fewer than 2 states: the candidate does
 * not depend on t); 1 every positive target nil (lambda_min > lambda_max, or lambda_min < 0, where the model is
 * invalid at the first evaluation); 2 rising; 3 not rising.  y_lo, y_hi, b1 and b2 are 0 for kinds 0 and 1.
 *
 * The bounds belong to the pair: srv_slo_* are not read (srv_has_target and the other gates decide kind 0), nor
 * are fleet->unlimited and the capacities.  Any column of out may be NULL (not written).  The fleet becomes
 * resident, and wva_summarize returns WVA_ERR_STATE afterwards.  WVA_ERR_BAD_ARG: out NULL.  WVA_ERR_UNSUPPORTED:
 * the queue-size rule, before any kernel is launched, as wva_analyze refuses it; a boundary solve whose rescale
 * loop does not terminate (wva_last_error names the pair and the end).
 */
typedef struct wva_slo_bounds_out {
    uint8_t *kind; /* [S*A*2] */
    float *y_lo;   /* [S*A*2] */
    float *y_hi;   /* [S*A*2] */
    float *b1;     /* [S*A*2] */
    float *b2;     /* [S*A*2] */
} wva_slo_bounds_out;
int wva_slo_bounds(wva_handle *h, const wva_fleet *fleet, wva_slo_bounds_out *out);

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
 * the most recent call with host results, and of the whole call's device work
 * (the *_device calls do not time themselves). */
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

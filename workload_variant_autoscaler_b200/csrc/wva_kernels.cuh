// wva_kernels.cuh — sm_90a kernels of the WVA optimizer hot path.
//
//   build_pair_tables   servRate[n] (+ double-word reciprocal) per (server, accelerator)
//   grid_* kernels K2   one Analyze per (server, acc, batch, replica) cell: row sharing, length-class
//                       sort, persistent warps pulling 32-cell items, fused feasibility + batch-rank minimum
//   grid_fallback       stored-vector re-run of the rare cells the streaming solve bails on
//   grid_finalize  K3   per-server argmin over partials (warp shuffle -> smem -> record)
//   trivial_kernel      nil / zero-load candidates (overloads: per level of wva_load_grid, wva_slo_grid and
//                       wva_workload_grid)
//   unlimited_kernel    Server.Calculate value + SolveUnlimited argmin per server (overload: per load level)
//   trace_kernel        the same tick by tick, each tick's winner the next tick's current allocation
//   profile_kernel      the profile grid's records per (level, pair) from the key records, priced at the level
//   profile_trace_kernel  the profile trace's records per (tick, pair), the tail's records priced at the tick
//   size_grid_finalize  the same over (accelerator x batch size) per server, one warp per server
//   sweep_kernel        Analyze over a rate sweep per (server, acc)
//
// K1, CreateAllocation per (server, accelerator) candidate (the rounds, the warp-per-candidate kernel and the
// stored-vector fallback), is in wva_size.cuh.
#pragma once
#include "wva_device.cuh"

namespace wva {

// The columns of wva_fleet in declaration order: X(wva_fleet member, DevFleet / HostFleet member, element type,
// length).  The length is A (accelerators), T (accelerator types), MA (models x accelerators) or S (servers).
// DevFleet and the host engine's copy, upload and NULL checks are generated from this list.  The host arena
// follows this order, and wva_update_load copies srv_arrival_rpm, srv_in_tokens and srv_out_tokens as one
// range: those three must stay adjacent.
#define WVA_FLEET_COLUMNS(X)                          \
    X(acc_cost, acc_cost, float, A)                   \
    X(acc_multiplicity, acc_mult, int32_t, A)         \
    X(acc_type, acc_type, int32_t, A)                 \
    X(type_capacity, type_capacity, int32_t, T)       \
    X(perf_present, perf_present, uint8_t, MA)        \
    X(perf_alpha, perf_alpha, float, MA)              \
    X(perf_beta, perf_beta, float, MA)                \
    X(perf_gamma, perf_gamma, float, MA)              \
    X(perf_delta, perf_delta, float, MA)              \
    X(perf_acc_count, perf_acc_count, int32_t, MA)    \
    X(perf_max_batch, perf_max_batch, int32_t, MA)    \
    X(perf_at_tokens, perf_at_tokens, int32_t, MA)    \
    X(srv_model, srv_model, int32_t, S)               \
    X(srv_priority, srv_priority, int32_t, S)         \
    X(srv_has_target, srv_has_target, uint8_t, S)     \
    X(srv_slo_itl, srv_slo_itl, float, S)             \
    X(srv_slo_ttft, srv_slo_ttft, float, S)           \
    X(srv_slo_tps, srv_slo_tps, float, S)             \
    X(srv_keep_acc, srv_keep_acc, uint8_t, S)         \
    X(srv_min_replicas, srv_min_replicas, int32_t, S) \
    X(srv_max_batch, srv_max_batch, int32_t, S)       \
    X(srv_arrival_rpm, srv_arrival_rpm, float, S)     \
    X(srv_in_tokens, srv_in_tokens, int32_t, S)       \
    X(srv_out_tokens, srv_out_tokens, int32_t, S)     \
    X(srv_cur_acc, srv_cur_acc, int32_t, S)           \
    X(srv_cur_replicas, srv_cur_replicas, int32_t, S) \
    X(srv_cur_cost, srv_cur_cost, float, S)

// Device image of wva_fleet (all pointers are device pointers).
struct DevFleet {
    int A, T, M, S;
#define WVA_DEV_COLUMN(abi, name, type, len) const type* name;
    WVA_FLEET_COLUMNS(WVA_DEV_COLUMN)
#undef WVA_DEV_COLUMN
    int ratio;      // config.MaxQueueToBatchRatio
    float penalty;  // config.AccelPenaltyFactor
};

// One candidate allocation (core.Allocation, pkg/core/allocation.go:13-24).
struct Cand {
    float value, cost;
    int replicas, batch, acc;
    float itl, ttft, rho, max_rate;
    int feasible;
};
__device__ __forceinline__ Cand cand_nil() {
    Cand c;
    c.value = 0.f; c.cost = 0.f; c.replicas = 0; c.batch = 0; c.acc = -1;
    c.itl = 0.f; c.ttft = 0.f; c.rho = 0.f; c.max_rate = 0.f; c.feasible = 0;
    return c;
}
// Grid winner order: value, cost, replicas, batch, accelerator id (ascending).
__device__ __forceinline__ bool cand_better(const Cand& x, const Cand& y) {
    if (!x.feasible) return false;
    if (!y.feasible) return true;
    if (x.value != y.value) return x.value < y.value;
    if (x.cost != y.cost) return x.cost < y.cost;
    if (x.replicas != y.replicas) return x.replicas < y.replicas;
    if (x.batch != y.batch) return x.batch < y.batch;
    return x.acc < y.acc;
}
__device__ __forceinline__ Cand cand_shfl_down(const Cand& c, int d) {
    Cand o;
    o.value = __shfl_down_sync(0xffffffffu, c.value, d);
    o.cost = __shfl_down_sync(0xffffffffu, c.cost, d);
    o.replicas = __shfl_down_sync(0xffffffffu, c.replicas, d);
    o.batch = __shfl_down_sync(0xffffffffu, c.batch, d);
    o.acc = __shfl_down_sync(0xffffffffu, c.acc, d);
    o.itl = __shfl_down_sync(0xffffffffu, c.itl, d);
    o.ttft = __shfl_down_sync(0xffffffffu, c.ttft, d);
    o.rho = __shfl_down_sync(0xffffffffu, c.rho, d);
    o.max_rate = __shfl_down_sync(0xffffffffu, c.max_rate, d);
    o.feasible = __shfl_down_sync(0xffffffffu, c.feasible, d);
    return o;
}
__device__ __forceinline__ Cand cand_warp_min(Cand c) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        Cand o = cand_shfl_down(c, d);
        if (cand_better(o, c)) c = o;
    }
    return c;
}

// The columns of wva_allocs in declaration order, each also a member of Cand: X(member, element type,
// required): wva_solve_greedy needs the required columns on input and reads a NULL column of the others as 0.
#define WVA_ALLOC_COLUMNS(X) \
    X(feasible, uint8_t, 1)  \
    X(acc, int32_t, 1)       \
    X(replicas, int32_t, 1)  \
    X(batch, int32_t, 0)     \
    X(cost, float, 1)        \
    X(value, float, 1)       \
    X(itl, float, 0)         \
    X(ttft, float, 0)        \
    X(rho, float, 0)         \
    X(max_rate, float, 0)

// SoA columns of wva_allocs on the device.
struct AllocCols {
#define WVA_ALLOC_COLUMN(name, type, required) type* name;
    WVA_ALLOC_COLUMNS(WVA_ALLOC_COLUMN)
#undef WVA_ALLOC_COLUMN
};
__device__ __forceinline__ void store_cand(const AllocCols& o, size_t i, const Cand& c) {
#define WVA_STORE_COLUMN(name, type, required) \
    if (o.name) o.name[i] = (type)c.name;
    WVA_ALLOC_COLUMNS(WVA_STORE_COLUMN)
#undef WVA_STORE_COLUMN
}
__device__ __forceinline__ Cand load_cand(const AllocCols& o, size_t i) {
    Cand c;
#define WVA_LOAD_COLUMN(name, type, required) c.name = o.name[i];
    WVA_ALLOC_COLUMNS(WVA_LOAD_COLUMN)
#undef WVA_LOAD_COLUMN
    return c;
}

// ---------------------------------------------------------------------------
// Gates of CreateAllocation (allocation.go:42-75) + candidate rule (server.go:70-82).
// bit0: the pair can be analysed under load; bit1: zero-load candidate; 0: nil.
// ---------------------------------------------------------------------------
enum { PAIR_LOAD = 1, PAIR_ZERO = 2 };

__device__ __forceinline__ int pair_class(const DevFleet& f, int s, int a, bool honour_keep) {
    if (honour_keep && f.srv_keep_acc[s] && f.srv_cur_acc[s] != -1 && f.srv_cur_acc[s] != a) return 0;
    if (f.srv_arrival_rpm[s] < 0.0f || f.srv_in_tokens[s] < 0 || f.srv_out_tokens[s] < 0) return 0;
    const int m = f.srv_model[s];
    if (m < 0 || m >= f.M) return 0;
    if (!f.perf_present[m * f.A + a]) return 0;
    if (!f.srv_has_target[s]) return 0;
    if (f.srv_arrival_rpm[s] == 0.0f || f.srv_out_tokens[s] == 0) return PAIR_ZERO;
    return PAIR_LOAD;
}
__device__ __forceinline__ int num_instances(const DevFleet& f, int m, int a) {  // model.go:50-57
    const int c = f.perf_acc_count[m * f.A + a];
    return c <= 0 ? 1 : c;
}
__device__ __forceinline__ QParams qparams_of(const DevFleet& f, int s, int a) {
    const int k = f.srv_model[s] * f.A + a;
    QParams q;
    q.alpha = f.perf_alpha[k]; q.beta = f.perf_beta[k]; q.gamma = f.perf_gamma[k]; q.delta = f.perf_delta[k];
    q.in_tok = f.srv_in_tokens[s]; q.out_tok = f.srv_out_tokens[s];
    return q;
}
__device__ __forceinline__ float total_rate_of(const DevFleet& f, int s) {  // allocation.go:134-139
    if (f.srv_slo_tps[s] == 0.0f) return __fdiv_rn(f.srv_arrival_rpm[s], 60.0f);
    return __fdiv_rn(f.srv_slo_tps[s], (float)f.srv_out_tokens[s]);
}
// ... at arrival rate rpm instead of the server's own (the load intervals' points are not in memory)
__device__ __forceinline__ float total_rate_of(const DevFleet& f, int s, float rpm) {
    if (f.srv_slo_tps[s] == 0.0f) return __fdiv_rn(rpm, 60.0f);
    return total_rate_of(f, s);
}
// The fleet as the load grid sees it at level l: the arrival rates are row l of the level list.
__device__ __forceinline__ DevFleet at_level(const DevFleet& f, const float* level_rpm, int l) {
    DevFleet fl = f;
    fl.srv_arrival_rpm = level_rpm + (size_t)l * f.S;
    return fl;
}
__device__ __forceinline__ float penalty_of(const DevFleet& f, int s, const Cand& c) {
    return transition_penalty(f.penalty, f.srv_cur_acc[s], f.srv_cur_replicas[s], f.srv_cur_cost[s], c.acc,
                              c.replicas, c.cost);
}
// zeroLoadAllocation: allocation.go:259-288 at batch size max_batch (value = cost; caller applies the penalty)
__device__ __forceinline__ Cand zero_load_alloc(const DevFleet& f, int s, int a, int max_batch) {
    Cand c = cand_nil();
    c.feasible = 1;
    const long long nrep = f.srv_min_replicas[s];
    if (nrep == 0) return c;  // accelerator "", all zero
    const int m = f.srv_model[s], k = m * f.A + a;
    const long long total = (long long)num_instances(f, m, a) * nrep;
    c.acc = a;
    c.replicas = (int)nrep;
    c.batch = max_batch;
    c.cost = __fmul_rn(f.acc_cost[a], (float)total);
    c.value = c.cost;
    c.itl = __fadd_rn(f.perf_alpha[k], f.perf_beta[k]);
    const float max_decode = __fadd_rn(f.perf_alpha[k], __fmul_rn(f.perf_beta[k], (float)max_batch));
    c.ttft = __fadd_rn(f.perf_gamma[k], f.perf_delta[k]);
    c.max_rate = __fdiv_rn((float)max_batch, __fadd_rn(c.ttft, max_decode));
    return c;
}
// ... at the batch size the server or the perf data fixes
__device__ __forceinline__ Cand zero_load_alloc(const DevFleet& f, int s, int a) {
    const int k = f.srv_model[s] * f.A + a;
    return zero_load_alloc(f, s, a, f.srv_max_batch[s] > 0 ? f.srv_max_batch[s] : f.perf_max_batch[k]);
}

// ---------------------------------------------------------------------------
// Shared head tables: entry n (0-based) of table t = {servRate[n], yh, yl} as doubles + {min(servRate[n..]),
// max(servRate[0..n])} as floats (32 B, two 16 B loads per head step), plus a float column
// ls[n] = sum_{i<n} log2(servRate[i]) used only to ESTIMATE chain lengths for scheduling.
// ---------------------------------------------------------------------------
// Per (table, batch index) constants shared by the 64 replica levels of a pair:
// x = RateRange.Max (req/s) for N = batch, y = log2 servRate[N-1], z = ls[N-1], w = log2 servRate[0].
// Per (server, replica index): x = rate (req/s), y = lambda (req/ms), z = log2 lambda.
__global__ void __launch_bounds__(128) build_pair_tables(DevFleet f, const int* __restrict__ tab_pair,
                                                         const long long* __restrict__ tab_off,
                                                         const int* __restrict__ tab_len, int n_tab,
                                                         double* __restrict__ tab, float* __restrict__ ls,
                                                         const int* __restrict__ batch, int B,
                                                         float4* __restrict__ pb) {
    __shared__ double wsum[4];
    __shared__ double carry_s;
    const int t = blockIdx.x;
    if (t >= n_tab) return;
    const int pair = tab_pair[t];
    const int s = pair / f.A, a = pair % f.A;
    const QParams q = qparams_of(f, s, a);
    double* out = tab + 4 * tab_off[t];
    const int len = tab_len[t];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* l = ls ? ls + tab_off[t] + t : nullptr;  // len + 1 entries per table
    // forward sweep in tiles of 128: entries + exclusive prefix sum of log2(servRate)
    if (threadIdx.x == 0) carry_s = 0.0;
    __syncthreads();
    for (int base = 0; base < len; base += blockDim.x) {
        const int n = base + threadIdx.x;
        double lg = 0.0;
        if (n < len) {
            const float srf = serv_rate(q, n + 1);
            const double sr = (double)srf;
            const Recip r = make_recip(sr);
            out[4 * n + 0] = sr;
            out[4 * n + 1] = r.yh;
            out[4 * n + 2] = r.yl;
            lg = (double)log2f(srf);
        }
        double inc = lg;  // inclusive warp scan
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const double o = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += o;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        double off = carry_s;
        for (int w = 0; w < warp; ++w) off += wsum[w];
        if (l && n < len) l[n] = (float)(off + inc - lg);
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry_s = off + inc;
        __syncthreads();
    }
    if (l && threadIdx.x == 0) l[len] = (float)carry_s;
    // column 4 = {float suffix minimum, float prefix maximum} of servRate (exact: the rates are float32).
    // A NaN rate poisons the suffix minimum to 0 (early exit disabled) and the prefix maximum to +inf.
    __shared__ float wmin[4];
    __shared__ float carry_m;
    if (threadIdx.x == 0) carry_m = 3.402823466e38f;
    __syncthreads();
    for (int base = 0; base < len; base += blockDim.x) {  // backward: suffix minimum
        const int n = len - 1 - (base + threadIdx.x);     // thread 0 takes the last entry
        float v = n >= 0 ? (float)out[4 * n] : 3.402823466e38f;
        if (!(v == v)) v = 0.0f;
        float m = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const float o = __shfl_up_sync(0xffffffffu, m, d);
            if (lane >= d) m = fminf(m, o);
        }
        if (lane == 31) wmin[warp] = m;
        __syncthreads();
        float pre = carry_m;
        for (int w = 0; w < warp; ++w) pre = fminf(pre, wmin[w]);
        m = fminf(m, pre);
        if (n >= 0) ((float*)(out + 4 * n + 3))[0] = m;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry_m = m;
        __syncthreads();
    }
    if (threadIdx.x == 0) carry_m = 0.0f;
    __syncthreads();
    for (int base = 0; base < len; base += blockDim.x) {  // forward: prefix maximum
        const int n = base + threadIdx.x;
        float v = n < len ? (float)out[4 * n] : 0.0f;
        if (!(v == v)) v = 3.402823466e38f;
        float m = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const float o = __shfl_up_sync(0xffffffffu, m, d);
            if (lane >= d) m = fmaxf(m, o);
        }
        if (lane == 31) wmin[warp] = m;
        __syncthreads();
        float pre = carry_m;
        for (int w = 0; w < warp; ++w) pre = fmaxf(pre, wmin[w]);
        m = fmaxf(m, pre);
        if (n < len) ((float*)(out + 4 * n + 3))[1] = m;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry_m = m;
        __syncthreads();
    }
    if (pb) {
        const float l2s0 = log2f((float)out[0]);
        for (int bi = threadIdx.x; bi < B; bi += blockDim.x) {
            const int b = batch[bi];
            const float sN = (float)out[4 * (b - 1)];
            pb[(size_t)t * B + bi] = make_float4(rate_max_of(sN), log2f(sN), l[b - 1], l2s0);
        }
    }
}


// ---------------------------------------------------------------------------
// K2: candidate grid.
//
//   grid_rows        per (pair, replica level): the chain every large-enough batch size shares
//                    (solve_row); also the (server, replica) rate block and the batch-rank reset
//   grid_order       per server: without a cell table, the rows' order under grid_finalize's key, the cells
//                    that share their row's chain up to the row's first feasible one and the server's bound
//                    (the smallest key of a feasible cell found); then the cells left for grid_kernel as two
//                    rank intervals per row, listed in chunks of at most 4096 of one pair
//   grid_sort_cands  per chunk (fixed grid, a chunk per CTA at a time): the per-cell gates, a log-domain length
//                    estimate, an 8-bit class and a local counting sort -> warp items; the last CTA plans
//                    grid_kernel's queues (grid_items_plan)
//   grid_items_scatter  items ordered globally, longest class first
//   grid_kernel      persistent CTA per SM; warps pull items (32 cells of nearly equal chain length)
//                    from a long and a short queue: streaming solve, metrics, SLO feasibility,
//                    per-cell columns, atomicMin of the smallest feasible batch rank per
//                    (server, accelerator, replica) and of the server's bound; an item whose cells
//                    are all above the bound by then is skipped
//   grid_fallback   stored-vector re-run of the rare cells the streaming solve bails on
//   grid_shared     with a cell table, per (pair, replica level): every cell that shares the row's chain
//   grid_finalize   per-server argmin (warp shuffle -> shared memory -> winner record)
//
// For a fixed (server, accelerator, replica level) the transition penalty and the cost do
// not depend on the batch size, so the winner among batch sizes is the smallest feasible
// one; the per-server winner is then the best of the A*R survivors under the order
// value, cost, replicas, batch, accelerator.
// ---------------------------------------------------------------------------
struct CellCols {
    uint8_t* flags;  // bit0: Analyze ok, bit1: SLO-feasible
    float *ttft, *itl, *rho, *throughput;
};
constexpr int kSortChunk = 8192;   // cells per CTA in the local counting sort
constexpr int kSortThreads = 512;
constexpr int kGridStash = 24;     // chain states kept in shared memory between the two passes (per lane)
constexpr int kClasses = 256;      // 8-bit length classes; class 255 = not analysable
struct GridArgs {
    DevFleet f;
    const int* batch;        // [B]
    const int* batch_rank;   // [B] rank of batch[bi] in ascending (batch, bi) order
    const int* rank_to_bi;   // [B] inverse of batch_rank
    const int* replicas;     // [R]
    int B, R;
    const double* tab;       // shared head tables
    const float* ls;         // prefix log2 sums (estimate only)
    const long long* pair_tab_off;  // [S*A] entry offset of the pair's table (-1: none)
    const int* pair_tab_idx;        // [S*A] table index (for the ls / pb columns)
    const float4* pb;               // [n_tab * B] per (table, batch): rmax, log2 sN, ls[N-1], log2 s0
    float4* rt;               // [S * R] per (server, replica): rate, lambda, log2 lambda
    double* row_acc;                // [S*A*R] shared-chain results per (server, accelerator, replica)
    double* row_sump;
    int* row_j;                     // last state of the shared chain (INT_MAX: no sharing)
    int Bmax;                       // table length
    long long n_cells;
    unsigned* order;         // [n_cells] cell ids, sorted by length class inside each of grid_order's chunks
    unsigned long long* items;         // warp work items (start | count << 32 | class << 40), unsorted
    unsigned long long* items_sorted;  // the same, longest class first
    unsigned* item_count;    // [0] number of items, [1..256] items per class, [257..512] class cursors
    int* best_rank;          // [S*A*R] smallest feasible batch rank (INT_MAX: none)
    CellCols cells;          // internal per-cell columns (ttft, itl, rho always present)
    float4* pair_rec;        // [S*A][3] per pair: {alpha, beta, gamma, delta}, {in_tok, out_tok (int bits), slo_ttft, slo_itl},
                             // {min_replicas, tps flag (int bits), 0, 0} -- one 48-byte record instead of ten scattered loads
    uint4* recs;             // [items][32] per sorted cell: {cell, lambda bits, table entry offset, batch size | class << 23 | pad << 31}
    int want_cells;          // 0: the caller did not ask for the cell table -> cells that share their row's chain store
                             // nothing and are evaluated only up to the row's first feasible one (grid_finalize
                             // recomputes the few winners among them), and cells that cannot be a server's winner
                             // are skipped (grid_order); 1: every cell is evaluated and stored
    int prune;               // grid_order ranks the rows (A <= 256, Bmax < 2^24, A*R <= kOrderMaxRows; want_cells == 0)
    unsigned* row_grp;       // [S*A*R] group rank of the row: rows of the server strictly below it in (value, cost, replicas)
    unsigned long long* bound;  // [S] smallest key of a feasible cell found so far (kBoundOff: no pruning)
    // cells that need the stored-vector fallback: an FbList's fields, kept flat so that the ints below keep their
    // parameter offsets (a nested FbList pads to 24 bytes)
    int* fb_count;
    unsigned long long* fb_cells;
    int fb_cap;
    int long_per_sm;         // grid_kernel: long items per sub-partition 0 (< 0: chosen per launch by grid_items_plan)
    int n_ctas;              // CTAs of grid_kernel (= SMs)
    int long_cls;            // items of class <= long_cls are "long" ...
    unsigned long_cap;       // ... up to this many (long_per_sm x CTAs)
    unsigned* dbg_cycles;    // diagnostics: per order index, SM cycles spent in grid_kernel (or NULL)
    size_t dbg_n;            // cells; dbg_cycles[dbg_n + idx] holds the warp timeline (start ns, SM, end ns)
    // grid_order -> grid_sort_cands: the cells handed to grid_kernel, row by row
    int4* row_cand;          // [S*A*R] {row's first candidate inside its pair, n1, s2, 0}: the row's candidates are the
                             // ranks [0, n1) and then s2, s2 + 1, ...
    uint4* chunks;           // chunk list: {pair, first candidate inside the pair, count, place in order[]}
};

// A cell's place in grid_finalize's order (value, cost, replicas, batch, accelerator) among the cells of its server:
// the row's group rank, then the batch SIZE (repeated sizes stay tied), then the accelerator.  A cell whose key is
// strictly above the key of some feasible cell of the same server cannot be the server's winner.
constexpr unsigned long long kBoundOff = ~0ull;       // the server is not pruned (no order, or a NaN value / cost)
constexpr unsigned long long kBoundNone = ~0ull - 1;  // no feasible cell found yet (above every key)
__device__ __forceinline__ unsigned long long cell_key(unsigned grp, int b, int a) {
    return ((unsigned long long)grp << 32) | ((unsigned long long)(unsigned)b << 8) | (unsigned)a;
}

__device__ __forceinline__ void decode_cell(const GridArgs& g, long long cell, int& s, int& a, int& bi, int& ri) {
    unsigned t = (unsigned)cell;  // n_cells < 2^32 (checked on the host): 32-bit divisions
    const unsigned R = (unsigned)g.R, B = (unsigned)g.B, A = (unsigned)g.f.A;
    unsigned q = t / R;
    ri = (int)(t - q * R);
    t = q;
    q = t / B;
    bi = (int)(t - q * B);
    t = q;
    q = t / A;
    a = (int)(t - q * A);
    s = (int)q;
}

// Estimated number of chain states before exact early termination (scheduling only; any
// value is correct, a good one makes the 32 lanes of a warp finish together).
__device__ __forceinline__ float estimate_len(const double* /*tab*/, const float* ls, int N, int K, float /*lambda*/,
                                              float l2lam, float l2s0, float l2sN, float lsNm1) {
    const float thr = -78.0f + fminf(0.0f, l2lam - l2s0);
    const float d = l2sN - l2lam;                     // tail decay per state (> 0 when analysable)
    const float L0 = (float)(N - 1) * l2lam - lsNm1;  // log2 p[N-1]
    float est;
    if (L0 >= thr || N == 1) {
        est = (float)(N - 1) + (L0 - thr) / fmaxf(d, 1e-9f) + 2.0f;
    } else {
        // the chain dies inside the head.  log2 p[j] = j*l2lam - ls[j] rises from 0 to the mode and
        // falls afterwards, and thr < 0, so {j : log2 p[j] < thr} is an upper set: one binary search
        int lo = 1, hi = N - 1;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((float)mid * l2lam - ls[mid] < thr) hi = mid; else lo = mid + 1;
        }
        est = (float)lo + 2.0f;
    }
    return fminf(fmaxf(est, 2.0f), (float)K);
}
__device__ __forceinline__ int length_class(float est) {  // 0 = longest ... 254 = shortest
    const int c = (int)(log2f(est) * 12.0f);  // ~6 % wide classes
    return 254 - min(max(c, 0), 254);
}

// Warp-aggregated shared-memory counter: returns this lane's slot among the lanes that
// increment the same counter (one atomic per distinct counter per warp).
__device__ __forceinline__ unsigned agg_inc(unsigned* counters, int key) {
    const unsigned peers = __match_any_sync(__activemask(), key);
    const int leader = __ffs(peers) - 1;
    const int lane = threadIdx.x & 31;
    unsigned base = 0;
    if (lane == leader) base = atomicAdd(&counters[key], (unsigned)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    return base + __popc(peers & ((1u << lane) - 1u));
}

// SLO feasibility of an analysed cell (the build's grid semantics, SURVEY.md §8d).  The per-server
// targets and the stability limit of the (pair, batch) are row constants; rate/1000 is the cell's lambda.
struct FeasRow {
    float slo_ttft, slo_itl, lim;  // lim = RateRange.Max/1000 * (1 - 0.1): Size's stability margin (queueanalyzer.go:231-234)
    int min_replicas;
    bool tps;
};
__device__ __forceinline__ float feas_lim(float rmax) { return __fmul_rn(__fdiv_rn(rmax, 1000.0f), __fsub_rn(1.0f, 0.1f)); }
__device__ __forceinline__ FeasRow feas_row(const DevFleet& f, int s, float rmax) {
    FeasRow fr;
    fr.slo_ttft = f.srv_slo_ttft[s];
    fr.slo_itl = f.srv_slo_itl[s];
    fr.min_replicas = f.srv_min_replicas[s];
    fr.tps = f.srv_slo_tps[s] > 0.0f;
    fr.lim = feas_lim(rmax);
    return fr;
}
__device__ __forceinline__ bool cell_feasible(const FeasRow& fr, int r, float lambda, const Metrics& m) {
    bool feas = (fr.slo_ttft == 0.0f || m.ttft <= fr.slo_ttft) && (fr.slo_itl == 0.0f || m.avg_token_time <= fr.slo_itl) &&
                (r >= fr.min_replicas);
    if (fr.tps) feas = feas && (lambda <= fr.lim);
    return feas;
}
__device__ __forceinline__ void store_cell(const GridArgs& g, long long cell, int ok, int feas, const Metrics& m) {
    g.cells.flags[cell] = (uint8_t)(ok | (feas << 1));
    g.cells.ttft[cell] = m.ttft;
    g.cells.itl[cell] = m.avg_token_time;
    g.cells.rho[cell] = m.rho;
    if (g.cells.throughput) g.cells.throughput[cell] = m.throughput;
}

// A cell that shares its row's chain (grid_shared): stats_from_row + metrics_from with everything that does
// not depend on the batch size hoisted — per pair (PairConst: the operands of EffectiveConcurrency, PrefillTime,
// DecodeTime), per (pair, replica level) (resp = avgNumInSystem / throughput, 1 - sumP).  Same operations in the
// same order on the same operands as the unhoisted functions, hence the same bits.
struct PairConst {
    float gamma, d_in, alpha, beta, ec_base, ec_den;
    int in_zero;
};
__device__ __forceinline__ PairConst pair_const(const QParams& q) {
    PairConst pc;
    const float tokens = (float)(q.out_tok - 1);                    // queueanalyzer.go:296-302
    pc.gamma = q.gamma;
    pc.alpha = q.alpha;
    pc.beta = q.beta;
    pc.d_in = __fmul_rn(q.delta, (float)q.in_tok);                  // delta * inTokens (:258, :300)
    pc.ec_base = __fadd_rn(q.gamma, __fmul_rn(q.alpha, tokens));
    pc.ec_den = __fadd_rn(pc.d_in, __fmul_rn(q.beta, tokens));
    pc.in_zero = q.in_tok == 0;
    return pc;
}
// resp: (float)acc / throughput with throughput = lambda * (1 - 0) = lambda
__device__ __forceinline__ float row_resp_time(double acc, float lambda) {
    return __fdiv_rn((float)acc, __fmul_rn(lambda, __fsub_rn(1.0f, 0.0f)));
}
__device__ __forceinline__ Metrics shared_cell_metrics(const PairConst& pc, double acc, double one_m_sump, float resp,
                                                       float lambda, int N) {
    const double in_serv = __dadd_rn(acc, __dmul_rn(one_m_sump, (double)N));  // mm1modelstatedependent.go:53
    const float in_serv_f = (float)in_serv;
    const float thr = __fmul_rn(lambda, __fsub_rn(1.0f, 0.0f));
    const float serv = __fdiv_rn(in_serv_f, thr);
    float w = __fsub_rn(resp, serv);
    if (w < 0.0f) w = 0.0f;
    const float fN = (float)N;
    const float eff = go_minf(go_maxf(__fdiv_rn(__fsub_rn(serv, pc.ec_base), pc.ec_den), 0.0f), fN);
    Metrics m;
    m.avg_prefill_time = pc.in_zero ? 0.0f : __fadd_rn(pc.gamma, __fmul_rn(pc.d_in, eff));
    m.avg_token_time = __fadd_rn(pc.alpha, __fmul_rn(pc.beta, eff));
    m.rho = go_minf(go_maxf(__fdiv_rn(in_serv_f, fN), 0.0f), 1.0f);
    m.throughput = __fmul_rn(thr, 1000.0f);
    m.avg_wait_time = w;
    m.ttft = __fadd_rn(w, m.avg_prefill_time);
    return m;
}

// The same evaluation when (float)avgNumInServers does not depend on the batch size.  avgNumInServers =
// acc + (1 - sumP) * N in float64, and 1 - sumP is a few ulps of 1 at most (the chain died before state N), so
// for all N <= Nmax the float64 value stays inside the float32 rounding interval of acc unless acc sits within
// ~1e-13 relative of an interval edge.  row_invariant() proves it for a (pair, replica level) with an exact bound:
// lo_b, hi_b = the float32 rounding boundaries around acc (exact in float64); |in_serv - acc| <= |m| N (1 + 2^-52)
// + acc 2^-53, and both distances are exact differences (Sterbenz), so d > 2 RN(|m| Nmax) + acc 2^-50 implies
// lo_b < in_serv < hi_b, i.e. (float)in_serv == (float)acc for every batch size of the grid.  Then the service
// time, the waiting time and the unclamped effective concurrency are constants of the row and a cell costs a
// min, two multiply-adds and the SLO comparisons.  Rows that fail the test take shared_cell_metrics.
struct RowInv {
    float f0, w0, effu;  // (float)avgNumInServers, waiting time, max(effective concurrency, 0) before the clamp at N
};
__device__ __forceinline__ bool row_invariant(const PairConst& pc, double acc, double one_m_sump, float resp, float lambda,
                                              int Nmax, RowInv& ri) {
    const float f0 = (float)acc;
    if (!(f0 > 1e-30f && f0 < 1e30f)) return false;
    const float up = __uint_as_float(__float_as_uint(f0) + 1u), dn = __uint_as_float(__float_as_uint(f0) - 1u);
    const double hi_b = 0.5 * ((double)f0 + (double)up), lo_b = 0.5 * ((double)dn + (double)f0);
    const double d = fmin(hi_b - acc, acc - lo_b);
    const double tb = __dmul_rn(fabs(one_m_sump), (double)Nmax);
    if (!(d > __dadd_rn(__dmul_rn(2.0, tb), __dmul_rn(acc, 0x1p-50)))) return false;
    const float thr = __fmul_rn(lambda, __fsub_rn(1.0f, 0.0f));
    const float serv = __fdiv_rn(f0, thr);
    float w = __fsub_rn(resp, serv);
    if (w < 0.0f) w = 0.0f;
    ri.f0 = f0;
    ri.w0 = w;
    ri.effu = go_maxf(__fdiv_rn(__fsub_rn(serv, pc.ec_base), pc.ec_den), 0.0f);
    return true;
}
__device__ __forceinline__ Metrics shared_cell_metrics_inv(const PairConst& pc, const RowInv& ri, float lambda, int N,
                                                           bool want_rho) {
    const float fN = (float)N;
    const float eff = go_minf(ri.effu, fN);
    Metrics m;
    m.avg_prefill_time = pc.in_zero ? 0.0f : __fadd_rn(pc.gamma, __fmul_rn(pc.d_in, eff));
    m.avg_token_time = __fadd_rn(pc.alpha, __fmul_rn(pc.beta, eff));
    m.rho = want_rho ? go_minf(go_maxf(__fdiv_rn(ri.f0, fN), 0.0f), 1.0f) : 0.0f;
    m.throughput = __fmul_rn(__fmul_rn(lambda, __fsub_rn(1.0f, 0.0f)), 1000.0f);
    m.avg_wait_time = ri.w0;
    m.ttft = __fadd_rn(ri.w0, m.avg_prefill_time);
    return m;
}

// One CTA per (server, accelerator) pair, one lane per replica level: the chain every large-enough
// batch size shares.  The pair's table is staged in shared memory first (coalesced), so the serial
// chains read it at shared-memory latency instead of waiting for L2 on every step.
constexpr int kRowsSmemEntries = 1536;  // 48 KB of 32-byte entries; longer tables are read from global
__global__ void __launch_bounds__(128) grid_rows(GridArgs g) {
    extern __shared__ double rows_tab[];
    const DevFleet& f = g.f;
    const int sa = blockIdx.x;
    const int s = sa / f.A;
    const long long toff = g.pair_tab_off[sa];
    const double* tab = toff >= 0 ? g.tab + 4 * toff : nullptr;
    const bool staged = toff >= 0 && g.Bmax <= kRowsSmemEntries;
    if (staged) {
        // all of a thread's loads first, then its stores: one L2 round trip instead of one per iteration
        const double2* src = (const double2*)tab;
        double2* dst = (double2*)rows_tab;
        const int n16 = 2 * g.Bmax;
        for (int i0 = threadIdx.x; i0 < n16; i0 += 8 * blockDim.x) {
            double2 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int i = i0 + u * blockDim.x;
                if (i < n16) v[u] = src[i];
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int i = i0 + u * blockDim.x;
                if (i < n16) dst[i] = v[u];
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {  // the pair's constants as one record (grid_kernel reads it once per item)
        const int a = sa - s * f.A;
        const int m = f.srv_model[s];
        float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m >= 0 && m < f.M) {
            const int k = m * f.A + a;
            r0 = make_float4(f.perf_alpha[k], f.perf_beta[k], f.perf_gamma[k], f.perf_delta[k]);
        }
        g.pair_rec[3 * sa + 0] = r0;
        g.pair_rec[3 * sa + 1] = make_float4(__int_as_float(f.srv_in_tokens[s]), __int_as_float(f.srv_out_tokens[s]),
                                             f.srv_slo_ttft[s], f.srv_slo_itl[s]);
        g.pair_rec[3 * sa + 2] = make_float4(__int_as_float(f.srv_min_replicas[s]),
                                             __int_as_float(f.srv_slo_tps[s] > 0.0f ? 1 : 0), 0.f, 0.f);
    }
    float l2s0 = 0.f, ls_end = 0.f;
    if (toff >= 0) {
        l2s0 = log2f((float)tab[0]);
        ls_end = (g.ls + toff + g.pair_tab_idx[sa])[g.Bmax - 1];
    }
    for (int ri = threadIdx.x; ri < g.R; ri += blockDim.x) {
        const size_t row = (size_t)sa * g.R + ri;
        int j = INT_MAX;
        double acc = 0.0, sump = 0.0;
        // per-replica rate, lambda and log2(lambda) of the server (rate = total / replicas, lambda = rate / 1000): every pair CTA
        // derives its own copy, the CTA of accelerator 0 publishes it for the later kernels; the
        // (pair, replica) slot of the batch-rank minimum is reset here too
        const float rate = __fdiv_rn(total_rate_of(f, s), (float)g.replicas[ri]);
        const float lambda = __fdiv_rn(rate, 1000.0f);
        const float4 rt = make_float4(rate, lambda, log2f(lambda), 0.0f);
        if (sa == s * f.A) g.rt[s * g.R + ri] = rt;
        g.best_rank[row] = INT_MAX;
        if (toff >= 0 && rt.x > 0.0f) {
            // skip rows whose chain is (by the log-domain estimate) still far from negligible at the end of
            // the table: they cannot be shared and would only burn Bmax steps to find that out
            const float thr = -78.0f + fminf(0.0f, rt.z - l2s0);
            const float Lend = (float)(g.Bmax - 1) * rt.z - ls_end;
            int jl = 0;
            if (Lend < thr + 8.0f) {
                const bool ok = staged ? solve_row(rows_tab, g.Bmax, rt.y, acc, sump, jl) : solve_row(tab, g.Bmax, rt.y, acc, sump, jl);
                if (ok) j = jl;
            }
        }
        g.row_j[row] = j;
        g.row_acc[row] = acc;
        g.row_sump[row] = sump;
    }
}

// Between grid_rows and grid_sort_cands: one CTA per server.  With a cell table (pruning off) only step 3 runs:
// grid_shared evaluates every shared cell after grid_kernel, which the walk of step 2 would only repeat.
//  1. Group ranks (g.prune): every (accelerator, replica level) row gets the number of rows of the server strictly
//     below it in (value, cost, replicas), with value and cost computed as grid_finalize computes them.  A counting
//     rank, Q threads per row.  It keeps key_better's order, ties included (-0 == +0); rows without a table take part
//     with a fixed key, which does not change the order of the others.  A NaN value or cost would make the order
//     depend on the reduction, so it turns pruning off for the server (bound = kBoundOff).
//  2. The shared runs (b >= jl + 2, K < 2^23): each row is walked from its first shared rank up to its first feasible
//     cell, which lowers best_rank; the smallest key among those cells is the server's bound.  Rows are taken in group
//     order, kOrderG lanes per row, and a row's walk also stops at the first cell whose key is above the bound so far
//     (keys grow along a row), so once a group has a feasible shared cell the rows of later groups stop at once.
//     A walk step is a chain of dependent loads, and a row without a feasible shared cell walks its whole run, so
//     the batch sizes in rank order and the pairs' RateRange.Max per rank are staged in shared memory first (in the
//     space the ranking used).
//  3. The candidates: the cells grid_sort_cands hands to grid_kernel, as rank intervals of each row.  Every rule that
//     drops a cell cuts a row at one rank, since batch sizes ascend with the rank: shared cells are the ranks
//     [lo, kK) (lo: the first rank with b >= jl + 2, B without sharing; kK: the first rank with K >= 2^23, the same
//     for every row), and cells above the bound the ranks [hi, B) (keys grow along a row).  So the candidates are
//     [0, min(lo, hi)) and [max(lo, kK), hi).  Rows with rt.x <= 0 and pairs without a table have none, nor, without
//     a cell table, do pairs with alpha > slo_itl (ITL = alpha + beta * eff >= alpha, eff >= 0, beta >= 0); with a
//     cell table grid_kernel stores their cells as analysed and not feasible.  A warp per pair scans its rows' counts
//     into their first candidates, then reserves the pair's chunks of kCandChunk candidates in the chunk list and
//     their places in order[] with one atomic.
//
// Without a cell table no pass over the shared cells is needed after grid_kernel.  Every cell that is never
// evaluated — a shared cell after the stop of its row's walk, or a non-shared cell that is not a candidate or that
// grid_sort_cands or grid_kernel skips — either cannot be feasible (the exact gates above and in grid_sort_cands) or
// has a key strictly above a feasible cell of its server.  So the winner W (the smallest key among the feasible cells)
// is evaluated, and so is every feasible cell of W's row below W, which has a smaller or equal key: best_rank of W's
// row is W's rank.  Any other best_rank is a feasible cell, whose key is >= W's.  grid_finalize picks W exactly as
// when every cell is evaluated.
constexpr int kOrderThreads = 1024, kOrderG = 4, kOrderMaxRows = 2048;
constexpr int kCandChunk = 4096;               // candidates per chunk of grid_sort_cands (never two pairs)
constexpr int kCandThreads = 256, kCandCtasPerSm = 4;
constexpr int kCandResv = 2 * kClasses + 16;   // item_count[kCandResv], [kCandResv + 1]: candidates, chunks reserved
__global__ void __launch_bounds__(kOrderThreads) grid_order(GridArgs g) {
    __shared__ float s_vc[2 * kOrderMaxRows];  // ranking: values | costs; walk: RateRange.Max per (accelerator, rank)
    __shared__ int s_rep[kOrderMaxRows];        // ranking: replicas; walk: batch size per rank
    float* s_val = s_vc;
    float* s_cost = s_vc + kOrderMaxRows;
    __shared__ unsigned s_grp[kOrderMaxRows];
    __shared__ unsigned short s_at[kOrderMaxRows];  // the row at each position of the group order
    __shared__ unsigned long long s_bound;
    const DevFleet& f = g.f;
    const int s = blockIdx.x, A = f.A, R = g.R, B = g.B, n = A * R;
    const size_t row0 = (size_t)s * n;
    const unsigned tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) s_bound = kBoundNone;
    int nan = 0;
    if (g.prune) {
        for (int k = tid; k < n; k += blockDim.x) {
            const int a = k / R, ri = k - a * R;
            float v = INFINITY, c = INFINITY;
            int r = INT_MAX;
            if (g.pair_tab_off[s * A + a] >= 0) {  // grid_finalize: cost, then value = penalty_of
                Cand x = cand_nil();
                x.acc = a;
                x.replicas = r = g.replicas[ri];
                x.cost = c = __fmul_rn(f.acc_cost[a], (float)((long long)num_instances(f, f.srv_model[s], a) * (long long)r));
                v = penalty_of(f, s, x);
                nan |= v != v || c != c;
            }
            s_val[k] = v;
            s_cost[k] = c;
            s_rep[k] = r;
        }
    }
    const bool prune = g.prune && !__syncthreads_or(nan);
    if (prune) {
        int q = 1;  // threads per row: a power of two <= 32, so that they are lanes of one warp
        while (q < 32 && 2 * q * n <= (int)blockDim.x) q *= 2;
        const int per = (int)blockDim.x / q;
        for (int base = 0; base < n; base += per) {
            const int i = base + (int)tid / q;
            unsigned lt = 0, eq = 0;  // rows strictly below row i; equal rows before it (its place among its ties)
            if (i < n) {
                const float vi = s_val[i], ci = s_cost[i];
                const int ri = s_rep[i];
                for (int j = (int)tid % q; j < n; j += q) {
                    const float vj = s_val[j], cj = s_cost[j];
                    const int rj = s_rep[j];
                    lt += vj < vi || (vj == vi && (cj < ci || (cj == ci && rj < ri)));
                    eq += vj == vi && cj == ci && rj == ri && j < i;
                }
            }
            for (int d = 1; d < q; d <<= 1) {
                lt += __shfl_xor_sync(0xffffffffu, lt, d);
                eq += __shfl_xor_sync(0xffffffffu, eq, d);
            }
            if (i < n && (int)tid % q == 0) {
                s_grp[i] = lt;
                s_at[lt + eq] = (unsigned short)i;
                g.row_grp[row0 + i] = lt;
            }
        }
    } else if (g.prune) {
        for (int k = tid; k < n; k += blockDim.x) g.row_grp[row0 + k] = 0;
    }
    __syncthreads();
    const bool stage_b = B <= kOrderMaxRows, stage_rmax = A * B <= 2 * kOrderMaxRows;
    if (stage_b)
        for (int r = tid; r < B; r += blockDim.x) s_rep[r] = g.batch[g.rank_to_bi[r]];
    if (stage_rmax)
        for (int k = tid; k < A * B; k += blockDim.x) {
            const int a = k / B, r = k - a * B;
            const long long toff = g.pair_tab_off[s * A + a];
            s_vc[k] = toff >= 0 ? g.pb[(size_t)g.pair_tab_idx[s * A + a] * B + g.rank_to_bi[r]].x : 0.0f;
        }
    __syncthreads();
    auto batch_at = [&](int r) { return stage_b ? s_rep[r] : g.batch[g.rank_to_bi[r]]; };
    const unsigned sub = lane % kOrderG, gmask = ((1u << kOrderG) - 1u) << (lane - sub);
    for (int base = 0; base < n && !g.want_cells; base += (int)blockDim.x / kOrderG) {
        const int p = base + (int)tid / kOrderG;
        const int k = p < n ? (prune ? s_at[p] : p) : 0;
        const int a = k / R, ri = k - a * R;
        const size_t row = row0 + k;
        const unsigned grp = prune ? s_grp[k] : 0u;
        const int jl = p < n ? g.row_j[row] : INT_MAX;  // a shared chain implies a table and a positive rate (grid_rows)
        int lo = 0;
        bool active = false;
        float4 rt;
        double acc, one_m_sump;
        float resp;
        PairConst pc;
        FeasRow fr;
        RowInv inv;
        int t, rep;
        bool is_inv;
        if (jl != INT_MAX) {
            int hi = B;  // first shared rank: the first rank whose batch size is >= jl + 2
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (batch_at(mid) < jl + 2) lo = mid + 1; else hi = mid;
            }
            active = lo < B;
        }
        if (active) {
            t = g.pair_tab_idx[s * A + a];
            rt = g.rt[s * R + ri];
            rep = g.replicas[ri];
            acc = g.row_acc[row];
            one_m_sump = __dsub_rn(1.0, g.row_sump[row]);
            resp = row_resp_time(acc, rt.y);
            pc = pair_const(qparams_of(f, s, a));
            fr = feas_row(f, s, 0.0f);
            is_inv = row_invariant(pc, acc, one_m_sump, resp, rt.y, g.Bmax, inv);
        }
        for (int r0 = lo; __any_sync(0xffffffffu, active); r0 += kOrderG) {
            const int r = r0 + (int)sub;
            bool feas = false, stop = false;
            unsigned long long key = 0;
            if (active && r < B) {
                const int b = batch_at(r);
                const int K = b + b * f.ratio;
                key = cell_key(grp, b, a);
                if (K >= (1 << 23) || (prune && key > *(volatile unsigned long long*)&s_bound)) {
                    stop = true;  // grid_kernel's cells from here on, or no cell from here on can win
                } else {
                    const float rmax = stage_rmax ? s_vc[a * B + r] : g.pb[(size_t)t * B + g.rank_to_bi[r]].x;
                    if (!(rt.x > rmax) && K >= 2) {  // Analyze: queueanalyzer.go:135-143
                        const Metrics m = is_inv ? shared_cell_metrics_inv(pc, inv, rt.y, b, false)
                                                 : shared_cell_metrics(pc, acc, one_m_sump, resp, rt.y, b);
                        if (fr.tps) fr.lim = feas_lim(rmax);
                        feas = cell_feasible(fr, rep, rt.y, m);
                    }
                }
            }
            const unsigned fm = __ballot_sync(0xffffffffu, feas) & gmask;
            const bool stopped = (__ballot_sync(0xffffffffu, stop) & gmask) != 0;
            if (fm && lane == (unsigned)(__ffs(fm) - 1)) {
                atomicMin(&g.best_rank[row], r);
                if (prune) atomicMin(&s_bound, key);
            }
            if (fm || stopped || r0 + kOrderG >= B) active = false;
        }
    }
    __syncthreads();
    const unsigned long long bound = prune ? s_bound : kBoundOff;
    if (tid == 0) g.bound[s] = bound;
    int kK = 0;  // the first rank with K >= 2^23
    for (int hi = B; kK < hi;) {
        const int mid = (kK + hi) >> 1, b = batch_at(mid);
        if (b + b * f.ratio < (1 << 23)) kK = mid + 1; else hi = mid;
    }
    for (int a = (int)(tid >> 5); a < A; a += kOrderThreads / 32) {
        const int sa = s * A + a;
        bool out = g.pair_tab_off[sa] < 0;
        if (!out && !g.want_cells) {  // a table implies a valid model index (pair_class == PAIR_LOAD)
            const int k = f.srv_model[s] * A + a;
            const float slo_itl = f.srv_slo_itl[s];
            out = slo_itl != 0.0f && f.perf_beta[k] >= 0.0f && f.perf_alpha[k] > slo_itl;
        }
        unsigned tot = 0;  // the pair's candidates
        for (int r0 = 0; r0 < R && !out; r0 += 32) {
            const int ri = r0 + (int)lane;
            const size_t row = (size_t)sa * R + ri;
            int n1 = 0, s2 = 0, cnt = 0;
            if (ri < R && !(g.rt[s * R + ri].x <= 0.0f)) {
                const int jl = g.row_j[row];
                int lo = B, hi = B;
                if (jl != INT_MAX) {
                    lo = 0;
                    for (int h = B; lo < h;) {
                        const int mid = (lo + h) >> 1;
                        if (batch_at(mid) < jl + 2) lo = mid + 1; else h = mid;
                    }
                }
                if (bound < kBoundNone) {  // only with prune: a key <= bound exists
                    const unsigned grp = s_grp[a * R + ri];
                    hi = 0;
                    for (int h = B; hi < h;) {
                        const int mid = (hi + h) >> 1;
                        if (cell_key(grp, batch_at(mid), a) > bound) h = mid; else hi = mid + 1;
                    }
                }
                n1 = min(lo, hi);
                s2 = max(lo, kK);
                cnt = n1 + max(hi - s2, 0);
            }
            int inc = cnt;
            for (int d = 1; d < 32; d <<= 1) {
                const int o = __shfl_up_sync(0xffffffffu, inc, d);
                if ((int)lane >= d) inc += o;
            }
            if (ri < R) g.row_cand[row] = make_int4((int)tot + inc - cnt, n1, s2, 0);
            tot += (unsigned)__shfl_sync(0xffffffffu, inc, 31);
        }
        if (tot) {
            const unsigned nch = (tot + kCandChunk - 1) / kCandChunk;
            unsigned long long at = 0;  // candidates reserved before this pair (low word), chunks (high word)
            if (lane == 0) at = atomicAdd((unsigned long long*)(g.item_count + kCandResv), (unsigned long long)nch << 32 | tot);
            at = __shfl_sync(0xffffffffu, at, 0);
            for (unsigned c = lane; c < nch; c += 32)
                g.chunks[(at >> 32) + c] = make_uint4((unsigned)sa, c * kCandChunk, min((unsigned)kCandChunk, tot - c * kCandChunk),
                                                      (unsigned)at + c * kCandChunk);
        }
    }
}

// Counter increment for lanes whose equal keys sit in CONTIGUOUS lane ranges (along a row the
// length class is monotone in the replica level, so equal classes are adjacent): one atomic per
// run instead of one per lane, found with a shuffle and a ballot.  Returns the lane's slot.
__device__ __forceinline__ unsigned seg_inc(unsigned* counters, int key) {
    const unsigned act = __activemask();
    const int lane = threadIdx.x & 31;
    const int prev = __shfl_up_sync(act, key, 1);
    const bool prev_active = lane > 0 && ((act >> (lane - 1)) & 1u);
    const unsigned heads = __ballot_sync(act, !prev_active || prev != key);
    const unsigned upto = (lane == 31) ? 0xffffffffu : ((2u << lane) - 1u);
    const int seg_start = 31 - __clz(heads & upto);
    const unsigned above = heads & ~upto;
    const int seg_end = above ? (__ffs(above) - 1) : 32;  // exclusive; inactive lanes start a new run too
    const unsigned seg_mask = (seg_end == 32 ? 0xffffffffu : ((1u << seg_end) - 1u)) & ~((1u << seg_start) - 1u) & act;
    unsigned base = 0;
    if (lane == seg_start) base = atomicAdd(&counters[key], (unsigned)__popc(seg_mask));
    base = __shfl_sync(act, base, seg_start);
    return base + __popc(seg_mask & ((1u << lane) - 1u));
}

// The end of a chunk's sort: cells[0, n) hold the chunk's cell ids, keys[0, n) their length classes (255: the cell
// is not handed to grid_kernel) and hist the class counts.  The counts are scanned into class cursors, the cells are
// scattered into order[obase ...] by class, and each run of 32 sorted cells becomes one warp work item tagged with
// its (longest) class.
__device__ __forceinline__ void sort_chunk_items(const GridArgs& g, const unsigned* cells, const uint8_t* keys,
                                                 uint8_t* sorted_keys, unsigned* hist, unsigned* cursor, int n,
                                                 unsigned obase) {
    __shared__ unsigned item_base;
    if (threadIdx.x < 32) {  // exclusive scan of the 256 class counts by one warp
        unsigned run = 0;
        for (int c0 = 0; c0 < kClasses; c0 += 32) {
            const unsigned v = hist[c0 + threadIdx.x];
            unsigned inc = v;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned o = __shfl_up_sync(0xffffffffu, inc, d);
                if ((int)threadIdx.x >= d) inc += o;
            }
            cursor[c0 + threadIdx.x] = run + inc - v;
            run += __shfl_sync(0xffffffffu, inc, 31);
        }
    }
    __syncthreads();
    const int n_active = (int)cursor[255];  // class 255 (not analysable) sorts last
    for (int k = threadIdx.x; k < n; k += kCandThreads) {
        const int key = keys[k];
        if (key == 255) continue;
        const unsigned pos = seg_inc(cursor, key);
        g.order[obase + pos] = cells[k];
        sorted_keys[pos] = (uint8_t)key;
    }
    const int n_items = (n_active + 31) >> 5;
    if (threadIdx.x == 0) item_base = n_items ? atomicAdd(g.item_count, (unsigned)n_items) : 0u;
    __syncthreads();
    for (int w = threadIdx.x; w < n_items; w += kCandThreads) {
        const unsigned start = obase + 32 * w;
        const unsigned cnt = (unsigned)min(32, n_active - 32 * w);
        const int cls = sorted_keys[32 * w];
        g.items[item_base + w] = (unsigned long long)start | ((unsigned long long)cnt << 32) |
                                 ((unsigned long long)cls << 40);
        agg_inc(g.item_count + 1, cls);  // global items-per-class histogram (warp-aggregated)
    }
}

// The last CTA of grid_sort_cands to get here turns the global histogram into class cursors and plans grid_kernel's
// queues (one launch less than a separate single-CTA kernel).
__device__ __forceinline__ void grid_items_plan(const GridArgs& g);
__device__ __forceinline__ void sort_plan_in_last_cta(const GridArgs& g) {
    __shared__ bool last_cta;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last_cta = atomicAdd(g.item_count + 2 * kClasses + 6, 1u) == gridDim.x - 1;
    __syncthreads();
    if (last_cta) {
        __threadfence();
        grid_items_plan(g);
    }
}

// grid_order's candidates, a chunk (at most kCandChunk candidates of one pair) per CTA at a time over a fixed grid.
// A candidate's replica level is the last row of the pair whose first candidate is at or before it, and its rank
// follows from that row's intervals.  The gates that grid_order's intervals leave to each cell — Analyze's
// RateRange.Max and K >= 2, and, without a cell table, TPS servers above the stability limit (with one, grid_kernel
// stores those cells as analysed and not feasible) — give class 255; the others get the length class, and
// sort_chunk_items sorts the chunk into items.  A chunk never holds two pairs, so neither does an item (grid_kernel
// fetches the pair record once per item).
__global__ void __launch_bounds__(kCandThreads) grid_sort_cands(GridArgs g) {
    __shared__ unsigned cells[kCandChunk];
    __shared__ uint8_t keys[kCandChunk];
    __shared__ uint8_t sorted_keys[kCandChunk];
    __shared__ unsigned hist[kClasses];
    __shared__ unsigned cursor[kClasses];
    const DevFleet& f = g.f;
    const int R = g.R, B = g.B;
    const unsigned n_chunks = g.item_count[kCandResv + 1];
    for (unsigned ci = blockIdx.x; ci < n_chunks; ci += gridDim.x) {
        const uint4 ch = g.chunks[ci];
        if (threadIdx.x < kClasses) hist[threadIdx.x] = 0;
        __syncthreads();
        const int sa = (int)ch.x, s = sa / f.A, t = g.pair_tab_idx[sa];
        const long long toff = g.pair_tab_off[sa];
        const bool tps = f.srv_slo_tps[s] > 0.0f && !g.want_cells;
        const int4* rc = g.row_cand + (size_t)sa * R;
        for (int k = threadIdx.x; k < (int)ch.z; k += kCandThreads) {
            const int j = (int)ch.y + k;
            int ri = 0;
            for (int hi = R - 1; ri < hi;) {
                const int mid = (ri + hi + 1) >> 1;
                if (rc[mid].x <= j) ri = mid; else hi = mid - 1;
            }
            const int4 row = rc[ri];
            const int q = j - row.x;
            const int bi = g.rank_to_bi[q < row.y ? q : row.z + (q - row.y)];
            const int b = g.batch[bi];
            const int K = b + b * f.ratio;
            const float4 rt = g.rt[s * R + ri];
            const float4 pb = g.pb[(size_t)t * B + bi];
            int key = 255;
            if (!(rt.x > pb.x) && K >= 2 && !(tps && !(rt.y <= feas_lim(pb.x))))  // Analyze: queueanalyzer.go:135-143
                key = length_class(estimate_len(g.tab + 4 * toff, g.ls + toff + t, b, K, rt.y, rt.z, pb.w, pb.y, pb.z));
            keys[k] = (uint8_t)key;
            cells[k] = ((unsigned)sa * (unsigned)B + (unsigned)bi) * (unsigned)R + (unsigned)ri;
            if (key != 255) seg_inc(hist, key);  // along a row, consecutive ranks: runs of equal classes
        }
        __syncthreads();
        sort_chunk_items(g, cells, keys, sorted_keys, hist, cursor, (int)ch.z, ch.w);
    }
    sort_plan_in_last_cta(g);
}

// Global order of the warp items by class (longest first): class cursors from the global
// histogram, then a multi-CTA scatter with warp-aggregated atomics.
// grid_kernel's CTA shape (the kernel is further down; grid_items_plan plans its queues)
#ifndef WVA_GK_WARPS
#define WVA_GK_WARPS 16
#endif
constexpr int kGkWarps = WVA_GK_WARPS;    // 4 per sub-partition; 128 registers per thread keep the two FP64 chains of pass 2 apart
constexpr int kGkThreads = kGkWarps * 32;
constexpr int kGkTabWin = 32;  // table entries staged per warp (solve_shared_t STAGED)
constexpr int kGkLong = -1;    // long-item warps per CTA: automatic     // long-item warps per SM (sub-partition 0)
// Model of grid_kernel's launch time, fitted on BASELINE config 2 with seeds 42..49 (tools/seed_times.py prints
// the plan next to the measured time): class c holds chains of 2^((254-c)/12) states;
//   item_us  what an item costs the short queue (two passes next to three other warps of the sub-partition,
//            stalls included): a cost per state + a fixed cost;
//   long_us  an item that has its sub-partition to itself: the same, without the sharing.
// The plan compares these times with each other only, so a clock that scales them all alike does not change it.
__device__ __forceinline__ float class_len(int c) { return exp2f((float)(254 - c) * (1.0f / 12.0f)); }
__device__ __forceinline__ float item_us(int c) { return 0.0987f * class_len(c) + 7.0f; }
__device__ __forceinline__ float long_us(int c) { return 0.0564f * class_len(c) + 4.0f; }
// Runs in ONE CTA of at least kClasses threads (the last CTA of the sort kernel to finish); threads beyond
// kClasses only take part in the barriers.
__device__ __forceinline__ void grid_items_plan(const GridArgs& g) {
    __shared__ unsigned cnt[kClasses + 1];  // exclusive prefix of the class counts (cnt[kClasses] = all items)
    __shared__ float wrk[kClasses + 1];     // exclusive prefix of the classes' work (warp-microseconds)
    __shared__ unsigned s_cnt[kClasses];
    __shared__ float s_wrk[kClasses];
    const int c = threadIdx.x;
    const bool on = c < kClasses;
    const unsigned mine = on ? __ldcg(g.item_count + 1 + c) : 0u;  // other CTAs' atomics: read at L2
    if (on) {
        s_cnt[c] = mine;
        s_wrk[c] = c < 255 ? (float)mine * item_us(c) : 0.0f;
    }
    __syncthreads();
    for (int d = 1; d < kClasses; d <<= 1) {  // inclusive Hillis-Steele scans
        const unsigned a = (on && c >= d) ? s_cnt[c - d] : 0u;
        const float w = (on && c >= d) ? s_wrk[c - d] : 0.0f;
        __syncthreads();
        if (on) {
            s_cnt[c] += a;
            s_wrk[c] += w;
        }
        __syncthreads();
    }
    if (on) {
        cnt[c + 1] = s_cnt[c];
        wrk[c + 1] = s_wrk[c];
        g.item_count[1 + kClasses + c] = s_cnt[c] - mine;  // class cursors for grid_items_scatter
    }
    if (c == 0) {
        cnt[0] = 0;
        wrk[0] = 0.0f;
    }
    __syncthreads();
    // grid_kernel's queues: the long queue is the head of the sorted list, the short queue the rest.
    // How many long items share a sub-partition (L) is chosen per launch from a two-term model of the
    // launch time, max(longest item at L per sub-partition, short-queue work / worker warps): more per
    // sub-partition slows the long chains (slow[] below, for L = 1..4) but
    // takes fewer sub-partitions away from the short queue.  Thread l evaluates L = l + 1.
    __shared__ float t_of[kGkWarps / 4];
    const int long_cls = g.long_cls < 0 ? -1 : (g.long_cls > 254 ? 254 : g.long_cls);
    const unsigned n_long_all = long_cls >= 0 ? cnt[long_cls + 1] : 0u;
    if (c < kGkWarps / 4) {
        const float slow[4] = {1.155f, 1.31f, 1.585f, 2.0f};
        const int l = c + 1;
        const unsigned nl = min(n_long_all, (unsigned)(l * g.n_ctas));
        const unsigned ctas = (nl + l - 1) / l;
        // work of the nl longest items: whole classes below the class that holds item nl, part of that one
        int lo = 0, hi = kClasses;  // first class k with cnt[k + 1] >= nl
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cnt[mid + 1] >= nl) hi = mid; else lo = mid + 1;
        }
        const int k = lo < kClasses ? lo : kClasses - 1;
        const float long_work = wrk[k] + (float)(nl - cnt[k]) * item_us(k);
        int c_max = 0;
        while (c_max < kClasses - 1 && cnt[c_max + 1] == 0) ++c_max;  // longest class present
        const float workers = (float)(kGkWarps * g.n_ctas) - (float)(kGkWarps / 4) * (float)ctas;
        const float t_short = (wrk[kClasses] - long_work) / fmaxf(workers, 1.0f);
        const float t_long = nl ? slow[c] * long_us(c_max) : 0.0f;
        t_of[c] = fmaxf(t_short, t_long);
        g.item_count[2 * kClasses + 8 + 2 * c] = __float_as_uint(t_short);  // diagnostics (wva_dbg_read_plan)
        g.item_count[2 * kClasses + 9 + 2 * c] = __float_as_uint(t_long);
    }
    __syncthreads();
    if (c == 0) {
        int L = g.long_per_sm;
        if (L < 0) {
            L = 1;
            for (int l = 2; l <= kGkWarps / 4; ++l)
                if (t_of[l - 1] < t_of[L - 1]) L = l;
        }
        const unsigned n_long = min(n_long_all, (unsigned)(L * g.n_ctas));
        g.item_count[2 * kClasses + 1] = n_long;
        g.item_count[2 * kClasses + 2] = 0;
        g.item_count[2 * kClasses + 3] = n_long;
        g.item_count[2 * kClasses + 4] = (unsigned)L;
    }
}
// Warp per item: the item takes its place in the global order (class cursors, longest class first) and its
// cells become 16-byte records in that order — cell id, lambda, the pair's table offset and the batch size —
// so that grid_kernel fetches an item's operands with ONE coalesced load instead of a chain of dependent ones
// (queue slot -> item -> order -> batch / replica / pair lists -> rate block).  A partial item (the last of a sort
// chunk) is padded with copies of its first cell, flagged, so that the whole warp takes part in the staged loads.
__global__ void __launch_bounds__(256) grid_items_scatter(GridArgs g) {
    const DevFleet& f = g.f;
    const unsigned n = *g.item_count;
    const unsigned lane = threadIdx.x & 31;
    const unsigned warps = (gridDim.x * blockDim.x) >> 5;
    for (unsigned i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const unsigned long long it = g.items[i];
        unsigned pos = 0;
        if (lane == 0) {
            pos = atomicAdd(g.item_count + 1 + kClasses + (unsigned)((it >> 40) & 0xff), 1u);
            g.items_sorted[pos] = it;
        }
        pos = __shfl_sync(0xffffffffu, pos, 0);
        const bool valid = lane < (unsigned)((it >> 32) & 0xff);
        const unsigned cell = g.order[(unsigned)it + (valid ? lane : 0u)];
        int s, a, bi, ri;
        decode_cell(g, (long long)cell, s, a, bi, ri);
        const float lambda = g.rt[s * g.R + ri].y;
        const unsigned toff = (unsigned)g.pair_tab_off[s * f.A + a];
        const unsigned b = (unsigned)g.batch[bi];
        // w: batch size (bits 0..22) | the item's length class (bits 23..30) | pad flag (bit 31)
        g.recs[(size_t)pos * 32 + lane] = make_uint4(cell, __float_as_uint(lambda), toff,
                                                     b | ((unsigned)((it >> 40) & 0xff) << 23) | (valid ? 0u : 0x80000000u));
    }
}

// ---------------------------------------------------------------------------
// grid_kernel — persistent, one CTA of kGkWarps warps per SM, warps pull items (32 cells of similar
// chain length) from two queues over the globally sorted item list:
//   * the LONG queue = the first n_long items (the longest chains, at most kGkLong per SM).  Their
//     latency bounds the launch: a 2816-state chain is 5632 dependent steps of several FP64 latencies, and
//     under equal sharing of a saturated FP64 pipe it would run 2-3x slower.  Warp w issues on SM
//     sub-partition w % 4 (tools/subpart_bench.cu), so the long items are pulled only by kGkLong
//     warps of sub-partition 0 and the other warps of that sub-partition stay parked until this
//     CTA's long warps are done: the long chains get a pipe to themselves;
//   * the SHORT queue = everything else, longest first, pulled by all other warps (and by the
//     sub-partition-0 warps once the CTA's long work is finished).
// ---------------------------------------------------------------------------
constexpr int kQLongN = 2 * kClasses + 1, kQLongCtr = kQLongN + 1, kQShortCtr = kQLongN + 2;  // in item_count[]

// Per-warp shared memory of grid_kernel (doubles): the pass-1 stash, the staged table window (+ the lanes' tail
// entries) and the pair record of the current item.
constexpr int kGkStashD = kGridStash * 32;              // [state][lane]
constexpr int kGkTbufD = kStagedTbufD;                  // staged table window + the lanes' tail entries
constexpr int kGkPairD = 8;                             // 48-byte pair record (padded to 64)
constexpr int kGkWarpD = kGkStashD + kGkTbufD + kGkPairD;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// One item: 32 records (one per lane) already in shared memory.  The solver gets everything it reads from the
// table in one batch of loads (solve_shared_t STAGED); the pair's constants travel into shared memory by
// cp.async meanwhile and are read back after the solve, so no operand of the epilogue is held in registers
// across the solver call and none is fetched by a dependent load afterwards.
__device__ __forceinline__ void item_run(const GridArgs& g, unsigned w, const uint4 rec, unsigned lane, double* warp_smem) {
    const DevFleet& f = g.f;
    double* stash_warp = warp_smem;
    double* tbuf_warp = warp_smem + kGkStashD;
    float4* pair_buf = reinterpret_cast<float4*>(warp_smem + kGkStashD + kGkTbufD);
    const unsigned idx = w * 32 + lane;
    const long long t_start = g.dbg_cycles ? clock64() : 0;
    unsigned long long t_start_ns = 0;
    if (g.dbg_cycles) asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t_start_ns));
    const unsigned cell = rec.x;
    const float lambda = __uint_as_float(rec.y);
    const double* tab = g.tab + 4 * (size_t)rec.z;
    const int N = (int)(rec.w & 0x7fffffu);
    const bool valid = (rec.w >> 31) == 0;
    const int K = N + N * f.ratio;
    const unsigned pair = cell / ((unsigned)g.B * (unsigned)g.R);
    if (g.prune) {
        // the bound may have dropped since grid_order (feasible cells found by earlier items): an item none of
        // whose cells can still be its server's winner is not solved
        const unsigned s = pair / (unsigned)f.A;
        const unsigned long long bound = __ldcg(g.bound + s);
        const unsigned grp = g.row_grp[(size_t)pair * g.R + cell % (unsigned)g.R];
        const bool live = valid && cell_key(grp, N, (int)(pair - s * (unsigned)f.A)) <= bound;
        if (!__any_sync(0xffffffffu, live)) return;
    }
    // an item holds one pair (a sort chunk never holds two, and a padded lane copies the item's first cell), so
    // lanes 0..2 fetch its record
    __syncwarp();  // the previous item's readers of pair_buf are done
    if (lane < 3) cp_async16(pair_buf + lane, g.pair_rec + 3 * (size_t)pair + lane);
    cp_async_commit();
    ModelStats st;
    const int rc = solve_shared_t<kGridStash, 10, true>(tab, N, K, lambda, st, stash_warp + lane, tbuf_warp);
    cp_async_wait<0>();
    __syncwarp();
    if (valid) {
        if (rc != kSolveOk) {
            fb_push(FbList{g.fb_count, g.fb_cells, g.fb_cap}, cell);
        } else {
            const float4 r0 = pair_buf[0], r1 = pair_buf[1], r2 = pair_buf[2];
            QParams q;
            q.alpha = r0.x; q.beta = r0.y; q.gamma = r0.z; q.delta = r0.w;
            q.in_tok = __float_as_int(r1.x); q.out_tok = __float_as_int(r1.y);
            FeasRow fr;
            fr.slo_ttft = r1.z;
            fr.slo_itl = r1.w;
            fr.min_replicas = __float_as_int(r2.x);
            fr.tps = __float_as_int(r2.y) != 0;
            fr.lim = feas_lim(rate_max_of(st.tail_rate));  // RateRange.Max of (pair, N) from servRate[N-1]
            int s, a, bi, ri;
            decode_cell(g, (long long)cell, s, a, bi, ri);
            const Metrics m = metrics_from(q, N, st);
            const bool feas = cell_feasible(fr, g.replicas[ri], lambda, m);
            store_cell(g, (long long)cell, 1, feas ? 1 : 0, m);
            if (feas) {
                atomicMin(&g.best_rank[(size_t)pair * g.R + ri], g.batch_rank[bi]);
                if (g.prune && __ldcg(g.bound + s) != kBoundOff)
                    atomicMin(g.bound + s, cell_key(g.row_grp[(size_t)pair * g.R + ri], N, a));
            }
            if (g.dbg_cycles) {
                g.dbg_cycles[idx] = (unsigned)(clock64() - t_start);
                if (lane < 3) {  // timeline: [0] start ns, [1] SM id, [2] end ns (low 32 bits of %globaltimer)
                    unsigned long long t_end;
                    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t_end));
                    unsigned smid;
                    asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
                    g.dbg_cycles[g.dbg_n + idx] = lane == 0 ? (unsigned)t_start_ns : lane == 1 ? smid : (unsigned)t_end;
                }
            }
        }
    }
    __syncwarp();
}

__global__ void __launch_bounds__(kGkThreads, 1) grid_kernel(GridArgs g) {
    extern __shared__ __align__(16) double grid_smem[];
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* warp_smem = grid_smem + (size_t)warp * kGkWarpD;
    const unsigned n_items = g.item_count[0], n_long = g.item_count[kQLongN];
    const bool sub0 = (warp & 3) == 0;
    // the long items are spread over as few CTAs as possible (long_per_sm per CTA): the other CTAs keep all
    // four sub-partitions for the short queue
    const int per = (int)g.item_count[kQLongN + 3];  // long items per sub-partition, chosen by grid_items_plan
    const int long_ctas = per > 0 ? (int)((n_long + per - 1) / per) : 0;
    const int my_long = (int)blockIdx.x < long_ctas ? per : 0;
    const bool long_warp = sub0 && (int)(warp >> 2) < my_long;
    // sub-partition 0: long_per_sm warps pull the long queue, the rest wait on named barrier 1 (blocked in
    // hardware: no issue slots) until the long warps of this CTA have drained the long queue
    const int n_parked = my_long > 0 ? kGkWarps / 4 - my_long : 0;
    const int bar_threads = 32 * (my_long + (n_parked > 0 ? n_parked : 0));
    if (long_warp && n_long) {
        for (;;) {
            unsigned w = 0;
            if (lane == 0) w = atomicAdd(g.item_count + kQLongCtr, 1u);
            w = __shfl_sync(0xffffffffu, w, 0);
            if (w >= n_long) break;
            const uint4 rec = g.recs[(size_t)w * 32 + lane];
            item_run(g, w, rec, lane, warp_smem);
        }
        if (n_parked > 0) asm volatile("bar.arrive 1, %0;" ::"r"(bar_threads) : "memory");
    } else if (sub0 && my_long > 0 && !long_warp) {
        asm volatile("bar.sync 1, %0;" ::"r"(bar_threads) : "memory");
    }
    // short queue: the list is longest-first and every warp takes the next item when it is free (LPT).  Reserving
    // items ahead of time (records prefetched two deep with cp.async) was measured and dropped: it hands a warp
    // two of the longest items back to back, and restricted to the short classes it bought nothing — the four
    // warps of a sub-partition already overlap each other's item boundaries.
    for (;;) {
        unsigned w = 0;
        if (lane == 0) w = atomicAdd(g.item_count + kQShortCtr, 1u);
        w = __shfl_sync(0xffffffffu, w, 0);
        if (w >= n_items) break;
        const uint4 rec = g.recs[(size_t)w * 32 + lane];
        item_run(g, w, rec, lane, warp_smem);
    }
}

// Stored-vector re-run of the cells grid_kernel bailed on (r.list holds cell ids).
__global__ void grid_fallback(GridArgs g, FbRun r) {
    const DevFleet& f = g.f;
    fb_rerun(r, [&](unsigned long long cell, double* p) {
        int s, a, bi, ri;
        decode_cell(g, (long long)cell, s, a, bi, ri);
        const int b = g.batch[bi], rep = g.replicas[ri];
        const double* tab = g.tab + 4 * g.pair_tab_off[s * f.A + a];
        const float rate = __fdiv_rn(total_rate_of(f, s), (float)rep);
        ModelStats st;
        const int rc = solve_stored(p, tab, b, b + b * f.ratio, __fdiv_rn(rate, 1000.0f), st);
        if (rc != 0) return rc;
        const Metrics m = metrics_from(qparams_of(f, s, a), b, st);
        const float rmax = rate_max_of((float)tab[4 * (b - 1)]);
        const bool feas = cell_feasible(feas_row(f, s, rmax), rep, __fdiv_rn(rate, 1000.0f), m);
        store_cell(g, (long long)cell, 1, feas ? 1 : 0, m);
        if (feas) atomicMin(&g.best_rank[((size_t)s * f.A + a) * g.R + ri], g.batch_rank[bi]);
        return 0;
    });
}

// With a cell table, the cells that share their row's chain (analysable, b >= jl + 2, K < 2^23), after grid_kernel
// and grid_fallback: every one is evaluated and stored.  Ranks ascend in batch size, so a row's shared cells are one
// run of ranks; its cells with K >= 2^23 (grid_kernel's) follow that run and end it.  (Without a cell table grid_order
// walks the shared runs before grid_kernel, up to each row's first feasible cell.)
//
// A warp owns 32 consecutive replica levels (coalesced stores) and one slice of kSharedSlice ranks; it finds which
// of its rows have shared cells in the slice, and each lane then walks one of those rows.
struct SharedRow {
    float4 rt;
    double acc, one_m_sump;
    float resp;
    PairConst pc;
    FeasRow fr;
    RowInv inv;
    int t, rep, lo, end;
    bool is_inv;
};
constexpr int kSharedThreads = 64, kSharedSlice = 32;
__global__ void __launch_bounds__(kSharedThreads) grid_shared(GridArgs g) {
    __shared__ SharedRow rows[kSharedThreads / 32][32];
    const DevFleet& f = g.f;
    const int R = g.R, B = g.B;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned wg = blockIdx.x * (kSharedThreads / 32) + warp;
    const unsigned n_slices = (unsigned)(B + kSharedSlice - 1) / kSharedSlice;
    const size_t my_row = (size_t)(wg / n_slices) * 32 + lane;
    const int r_beg = (int)(wg % n_slices) * kSharedSlice, r_end = min(B, r_beg + kSharedSlice);
    bool todo = false;
    if (my_row < (size_t)f.S * f.A * R) {
        const size_t row = my_row;
        const int jl = g.row_j[row];  // a shared chain implies a table and a positive rate (grid_rows)
        SharedRow& x = rows[warp][lane];
        x.lo = 0;
        x.end = r_end;
        if (jl != INT_MAX) {
            int hi = x.end;  // first shared rank: the first rank whose batch size is >= jl + 2
            while (x.lo < hi) {
                const int mid = (x.lo + hi) >> 1;
                if (g.batch[g.rank_to_bi[mid]] < jl + 2) x.lo = mid + 1; else hi = mid;
            }
            x.lo = max(x.lo, r_beg);
            todo = x.lo < x.end;
        }
        if (todo) {
            const unsigned sa = (unsigned)(row / R);
            const int ri = (int)(row - (size_t)sa * R), s = (int)(sa / f.A);
            x.t = g.pair_tab_idx[sa];
            x.rt = g.rt[s * R + ri];
            x.rep = g.replicas[ri];
            x.acc = g.row_acc[row];
            x.one_m_sump = __dsub_rn(1.0, g.row_sump[row]);
            x.resp = row_resp_time(x.acc, x.rt.y);
            x.pc = pair_const(qparams_of(f, s, (int)(sa - (unsigned)s * f.A)));
            x.fr = feas_row(f, s, 0.0f);
            x.is_inv = row_invariant(x.pc, x.acc, x.one_m_sump, x.resp, x.rt.y, g.Bmax, x.inv);
        }
    }
    __syncwarp();
    const unsigned own = __fns(__ballot_sync(0xffffffffu, todo), 0, (int)lane + 1);  // this lane's row (>= 32: none)
    bool active = own < 32;
    SharedRow x = rows[warp][active ? own : 0];
    const size_t row = __shfl_sync(0xffffffffu, my_row, active ? own : 0);
    const unsigned sa = (unsigned)(row / R);
    const int ri = (int)(row - (size_t)sa * R);
    bool found = false;  // this row's best_rank has been lowered
    for (int r = x.lo; active; ++r) {
        const int bi = g.rank_to_bi[r];
        const int b = g.batch[bi];
        const int K = b + b * f.ratio;
        if (K >= (1 << 23)) break;
        const float4 pb = g.pb[(size_t)x.t * B + bi];
        if (!(x.rt.x > pb.x) && K >= 2) {  // Analyze: queueanalyzer.go:135-143
            // the whole solve is shared with the row: only the N-dependent tail is per cell
            const Metrics m = x.is_inv ? shared_cell_metrics_inv(x.pc, x.inv, x.rt.y, b, true)
                                       : shared_cell_metrics(x.pc, x.acc, x.one_m_sump, x.resp, x.rt.y, b);
            if (x.fr.tps) x.fr.lim = feas_lim(pb.x);
            const bool feas = cell_feasible(x.fr, x.rep, x.rt.y, m);
            store_cell(g, ((long long)sa * B + bi) * R + ri, 1, feas ? 1 : 0, m);
            if (feas && !found) atomicMin(&g.best_rank[row], r);
            found = found || feas;
        }
        if (r + 1 >= x.end) active = false;
    }
}

// K3: per-server argmin.  One CTA per server: one candidate per (accelerator, replica
// level) = its smallest feasible batch size; warp-shuffle reduction, cross-warp reduction
// staged through shared memory.  The order (value, cost, replicas, batch, accelerator) does not involve the
// latency metrics, so only the keys are reduced; the winner's itl / ttft / rho are fetched once at the end:
// from the cell columns, or — for a cell that shares its row's chain and was not stored (want_cells == 0) —
// by the same stats_from_row + metrics_from evaluation grid_order ran for it.
struct GridKey {
    float value, cost;
    int replicas, batch, acc, bi, ri, feasible;  // bi < 0: zero-load allocation of accelerator ri
};
__device__ __forceinline__ bool key_better(const GridKey& x, const GridKey& y) {
    if (!x.feasible) return false;
    if (!y.feasible) return true;
    if (x.value != y.value) return x.value < y.value;
    if (x.cost != y.cost) return x.cost < y.cost;
    if (x.replicas != y.replicas) return x.replicas < y.replicas;
    if (x.batch != y.batch) return x.batch < y.batch;
    return x.acc < y.acc;
}
__device__ __forceinline__ GridKey key_warp_min(GridKey c) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        GridKey o;
        o.value = __shfl_down_sync(0xffffffffu, c.value, d);
        o.cost = __shfl_down_sync(0xffffffffu, c.cost, d);
        o.replicas = __shfl_down_sync(0xffffffffu, c.replicas, d);
        o.batch = __shfl_down_sync(0xffffffffu, c.batch, d);
        o.acc = __shfl_down_sync(0xffffffffu, c.acc, d);
        o.bi = __shfl_down_sync(0xffffffffu, c.bi, d);
        o.ri = __shfl_down_sync(0xffffffffu, c.ri, d);
        o.feasible = __shfl_down_sync(0xffffffffu, c.feasible, d);
        if (key_better(o, c)) c = o;
    }
    return c;
}
__global__ void __launch_bounds__(256) grid_finalize(GridArgs g, AllocCols winners) {
    const DevFleet& f = g.f;
    const int s = blockIdx.x;
    GridKey best{};
    best.acc = -1;
    for (int k = threadIdx.x; k < f.A * g.R; k += blockDim.x) {
        const int a = k / g.R, ri = k % g.R;
        const int rank = g.best_rank[((size_t)s * f.A + a) * g.R + ri];
        if (rank == INT_MAX) continue;
        const int bi = g.rank_to_bi[rank];
        const int r = g.replicas[ri];
        Cand c = cand_nil();
        const long long total = (long long)num_instances(f, f.srv_model[s], a) * (long long)r;
        c.acc = a;
        c.replicas = r;
        c.cost = __fmul_rn(f.acc_cost[a], (float)total);
        GridKey key;
        key.value = penalty_of(f, s, c);
        key.cost = c.cost;
        key.replicas = r;
        key.batch = g.batch[bi];
        key.acc = a;
        key.bi = bi;
        key.ri = ri;
        key.feasible = 1;
        if (key_better(key, best)) best = key;
    }
    // zero-traffic servers: the reference's zeroLoadAllocation per candidate accelerator
    for (int a = threadIdx.x; a < f.A; a += blockDim.x) {
        if (pair_class(f, s, a, true) == PAIR_ZERO) {
            Cand c = zero_load_alloc(f, s, a);
            GridKey key;
            key.value = penalty_of(f, s, c);
            key.cost = c.cost;
            key.replicas = c.replicas;
            key.batch = c.batch;
            key.acc = c.acc;
            key.bi = -1;
            key.ri = a;
            key.feasible = 1;
            if (key_better(key, best)) best = key;
        }
    }
    best = key_warp_min(best);
    __shared__ GridKey sm[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) sm[warp] = best;
    __syncthreads();
    if (warp == 0) {
        GridKey k = sm[0];
        if (lane > 0 && lane < (int)(blockDim.x >> 5)) k = sm[lane];
        if (lane >= (int)(blockDim.x >> 5)) k.feasible = 0;
        k = key_warp_min(k);
        if (lane == 0) {
            Cand c = cand_nil();
            if (k.feasible && k.bi < 0) {
                c = zero_load_alloc(f, s, k.ri);
                c.value = penalty_of(f, s, c);
            } else if (k.feasible) {
                const int a = k.acc, ri = k.ri, b = k.batch;
                c.feasible = 1;
                c.acc = a;
                c.replicas = k.replicas;
                c.batch = b;
                c.cost = k.cost;
                c.value = k.value;
                const size_t row = ((size_t)s * f.A + a) * g.R + ri;
                const long long cell = ((long long)row / g.R * g.B + k.bi) * g.R + ri;
                const int jl = g.row_j[row];
                const int K = b + b * f.ratio;
                if (!g.want_cells && jl != INT_MAX && b >= jl + 2 && K < (1 << 23)) {
                    // the cell shares its row's chain and was not stored: grid_order's evaluation again
                    const float lambda = g.rt[s * g.R + ri].y;
                    ModelStats st;
                    stats_from_row(g.row_acc[row], g.row_sump[row], b, lambda, st);
                    const Metrics m = metrics_from(qparams_of(f, s, a), b, st);
                    c.itl = m.avg_token_time;
                    c.ttft = m.ttft;
                    c.rho = m.rho;
                } else {
                    c.itl = g.cells.itl[cell];
                    c.ttft = g.cells.ttft[cell];
                    c.rho = g.cells.rho[cell];
                }
                c.max_rate = __fdiv_rn(rate_max_of((float)g.tab[4 * (g.pair_tab_off[s * f.A + a] + b - 1)]), 1000.0f);
            }
            store_cand(winners, s, c);
        }
    }
}

// nil and zero-load candidates (everything the size kernel does not own).  batch == NULL: one candidate per pair
// at the pair's own batch size; else B candidates per pair, record pair * B + bi at batch size batch[bi]
// (S * A * B < 2^31, checked on the host).
__global__ void trivial_kernel(DevFleet f, AllocCols cand, const int* batch, int B) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= f.S * f.A * B) return;
    const int pair = i / B, bi = i - pair * B;
    const int s = pair / f.A, a = pair % f.A;
    const int cls = pair_class(f, s, a, true);
    if (cls == PAIR_LOAD) return;
    Cand c = cand_nil();
    if (cls == PAIR_ZERO) c = batch ? zero_load_alloc(f, s, a, batch[bi]) : zero_load_alloc(f, s, a);
    store_cand(cand, i, c);
}
// ... of the load grid: L level blocks of S * A records (record l * S * A + pair), each pair classed at its
// level's rate level_rpm[l * S + s]; a zero-load candidate at the pair's own batch size (S * A * L < 2^31, checked
// on the host).
__global__ void trivial_kernel(DevFleet f, AllocCols cand, const float* level_rpm, int L) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_pairs = f.S * f.A;
    if (i >= n_pairs * L) return;
    const int l = i / n_pairs, pair = i - l * n_pairs;
    const int s = pair / f.A, a = pair % f.A;
    const int cls = pair_class(at_level(f, level_rpm, l), s, a, true);
    if (cls == PAIR_LOAD) return;
    store_cand(cand, i, cls == PAIR_ZERO ? zero_load_alloc(f, s, a) : cand_nil());
}
// ... of the SLO grid: L level blocks of S * A records (record l * S * A + pair); a pair's class and its nil or
// zero-load record read no target, so every block gets the same (S * A * L < 2^31, checked on the host).
__global__ void trivial_kernel(DevFleet f, AllocCols cand, int L) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_pairs = f.S * f.A;
    if (i >= n_pairs * L) return;
    const int pair = i % n_pairs;
    const int s = pair / f.A, a = pair % f.A;
    const int cls = pair_class(f, s, a, true);
    if (cls == PAIR_LOAD) return;
    store_cand(cand, i, cls == PAIR_ZERO ? zero_load_alloc(f, s, a) : cand_nil());
}
// ... of the workload grid: L level blocks of S * A records (record l * S * A + pair), each pair classed at its
// level's rate and tokens (row l of level_rpm, level_in and level_out); a zero-load candidate reads no tokens
// (S * A * L < 2^31, checked on the host).
__global__ void trivial_kernel(DevFleet f, AllocCols cand, const float* level_rpm, const int* level_in,
                               const int* level_out, int L) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_pairs = f.S * f.A;
    if (i >= n_pairs * L) return;
    const int l = i / n_pairs, pair = i - l * n_pairs;
    const int s = pair / f.A, a = pair % f.A;
    DevFleet fl = at_level(f, level_rpm, l);
    fl.srv_in_tokens = level_in + (size_t)l * f.S;
    fl.srv_out_tokens = level_out + (size_t)l * f.S;
    const int cls = pair_class(fl, s, a, true);
    if (cls == PAIR_LOAD) return;
    store_cand(cand, i, cls == PAIR_ZERO ? zero_load_alloc(f, s, a) : cand_nil());
}

// The columns of c from record i on.
__device__ __forceinline__ AllocCols cols_at(const AllocCols& c, size_t i) {
    AllocCols o;
#define WVA_OFFSET_COLUMN(name, type, required) o.name = c.name ? c.name + i : nullptr;
    WVA_ALLOC_COLUMNS(WVA_OFFSET_COLUMN)
#undef WVA_OFFSET_COLUMN
    return o;
}

// Server.Calculate's value (server.go:60-63) + SolveUnlimited (solver.go:63-79):
// one thread per server; strict '<' from MaxFloat32, lowest accelerator id wins ties.
__device__ __forceinline__ void unlimited_server(const DevFleet& f, const AllocCols& cand, const AllocCols& winners,
                                                 int s) {
    float min_val = 3.40282346638528859811704183484516925440e+38f;
    Cand best = cand_nil();
    for (int a = 0; a < f.A; ++a) {
        const size_t i = (size_t)s * f.A + a;
        if (!cand.feasible[i]) continue;
        Cand c = load_cand(cand, i);
        c.value = penalty_of(f, s, c);
        cand.value[i] = c.value;
        if (c.value < min_val) {
            min_val = c.value;
            best = c;
        }
    }
    store_cand(winners, s, best);
}
__global__ void unlimited_kernel(DevFleet f, AllocCols cand, AllocCols winners) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= f.S) return;
    unlimited_server(f, cand, winners, s);
}
// ... over the load grid's L level blocks (candidates l * S * A .., winners l * S ..); grid.y strides the levels.
__global__ void unlimited_kernel(DevFleet f, AllocCols cand, AllocCols winners, int L) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= f.S) return;
    for (int l = blockIdx.y; l < L; l += gridDim.y)
        unlimited_server(f, cols_at(cand, (size_t)l * f.S * f.A), cols_at(winners, (size_t)l * f.S), s);
}

// The workload trace's chain (DESIGN.md §3.13): one thread per server walks the L tick blocks (candidates
// (t * S + s) * A + a, winners t * S + s) with the current allocation c_t in registers, c_0 from the fleet.  The
// records hold CreateAllocation without the keepAccelerator mask, which does not read c_t.  Per tick: a pair the
// mask excludes against c_t's accelerator gets a nil record (sized or not), every other feasible record gets
// value = TransitionPenalty(c_t, .), winner t is SolveUnlimited's minimum (strict '<' from MaxFloat32, ties to the
// lower accelerator id), and c_{t+1} is the winner's (acc, replicas, cost) when it is feasible, c_t otherwise
// (Server.ApplyDesiredAlloc).
__global__ void trace_kernel(DevFleet f, AllocCols cand, AllocCols winners, int L) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= f.S) return;
    const bool keep = f.srv_keep_acc[s] != 0;
    int cur_acc = f.srv_cur_acc[s], cur_replicas = f.srv_cur_replicas[s];
    float cur_cost = f.srv_cur_cost[s];
    for (int t = 0; t < L; ++t) {
        float min_val = 3.40282346638528859811704183484516925440e+38f;
        Cand best = cand_nil();
        for (int a = 0; a < f.A; ++a) {
            const size_t i = ((size_t)t * f.S + s) * f.A + a;
            if (keep && cur_acc != -1 && cur_acc != a) {  // pair_class's keepAccelerator rule at c_t
                store_cand(cand, i, cand_nil());
                continue;
            }
            if (!cand.feasible[i]) continue;
            Cand c = load_cand(cand, i);
            c.value = transition_penalty(f.penalty, cur_acc, cur_replicas, cur_cost, c.acc, c.replicas, c.cost);
            cand.value[i] = c.value;
            if (c.value < min_val) {
                min_val = c.value;
                best = c;
            }
        }
        store_cand(winners, (size_t)t * f.S + s, best);
        if (best.feasible) {
            cur_acc = best.acc;
            cur_replicas = best.replicas;
            cur_cost = best.cost;
        }
    }
}

// The profile grid's records (DESIGN.md §3.14): L level blocks of S * A records (record (l * S + s) * A + a), one
// thread per record.  f_l is f with acc_cost and the perf_* columns of row l (profile_at).  A pair is classed at f_l:
// nil, zeroLoadAllocation at f_l, or, under load, the record its key was sized to on the key fleet (the row's
// alpha .. delta and N), with cost = acc_cost_l[a] * NumInstances_l * replicas, the only field that reads the row's
// cost or AccCount (S * A * L < 2^31, checked on the host).
struct ProfileArgs {
    DevFleet f;           // the resident fleet
    DevFleet rows;        // acc_cost and perf_* at level 0: the caller's row lists, or the fleet's own columns ...
    unsigned per_level;   // ... bit c (0: acc_cost, 1 .. 8: perf_* in list order) set: column c is a row list
    const int* rank;      // [L * M * A] the row's index among the distinct rows of (m, a); NULL: 0 everywhere
    const int* pair_off;  // [S * A] the pair's first entry in key_of, one entry per distinct row of (m, a)
    const int* key_of;    // the key record of (pair, row index); read only where the pair is a load
    AllocCols key;        // the key fleet's records
    AllocCols cand;       // [L * S * A]
    int L;
};
__device__ __forceinline__ DevFleet profile_at(const ProfileArgs& g, int l) {
    DevFleet fl = g.f;
    const size_t ra = (size_t)l * g.f.A, rma = (size_t)l * g.f.M * g.f.A;
    fl.acc_cost = g.rows.acc_cost + (g.per_level & 1u ? ra : 0);
#define WVA_PROFILE_ROW(name, bit) fl.name = g.rows.name + (g.per_level >> bit & 1u ? rma : 0);
    WVA_PROFILE_ROW(perf_present, 1)
    WVA_PROFILE_ROW(perf_alpha, 2)
    WVA_PROFILE_ROW(perf_beta, 3)
    WVA_PROFILE_ROW(perf_gamma, 4)
    WVA_PROFILE_ROW(perf_delta, 5)
    WVA_PROFILE_ROW(perf_acc_count, 6)
    WVA_PROFILE_ROW(perf_max_batch, 7)
    WVA_PROFILE_ROW(perf_at_tokens, 8)
#undef WVA_PROFILE_ROW
    return fl;
}
// A load record sized at another price or AccCount, priced at fl: cost = acc_cost[a] * NumInstances(m, a) *
// replicas and value = cost, the only fields of CreateAllocation that read either.
__device__ __forceinline__ Cand priced_at(const DevFleet& fl, int m, int a, Cand c) {
    if (c.feasible) {
        c.cost = __fmul_rn(fl.acc_cost[a], (float)((long long)num_instances(fl, m, a) * (long long)c.replicas));
        c.value = c.cost;
    }
    return c;
}
__global__ void profile_kernel(ProfileArgs g) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_pairs = g.f.S * g.f.A;
    if (i >= n_pairs * g.L) return;
    const int l = i / n_pairs, pair = i - l * n_pairs;
    const int s = pair / g.f.A, a = pair % g.f.A;
    const DevFleet fl = profile_at(g, l);
    const int cls = pair_class(fl, s, a, true);
    Cand c = cand_nil();
    if (cls == PAIR_ZERO) {
        c = zero_load_alloc(fl, s, a);
    } else if (cls == PAIR_LOAD) {
        const int m = fl.srv_model[s];
        const int j = g.rank ? g.rank[((size_t)l * fl.M + m) * fl.A + a] : 0;
        c = priced_at(fl, m, a, load_cand(g.key, g.key_of[g.pair_off[pair] + j]));
    }
    store_cand(g.cand, i, c);
}

// The profile trace's records (DESIGN.md §3.15): L tick blocks of S * A records (record (t * S + s) * A + a), one
// thread per record, after the workload grid's tail wrote every load pair's record in place at the key fleet's
// price.  f_t is f with row t of the load rows and of the profile rows (profile_at).  A pair is classed at f_t: nil,
// zeroLoadAllocation at f_t, or the tail's record priced at row t.  f carries keepAccelerator on the pinned servers
// only, whose pairs the tail did not size; trace_kernel applies the rest of the mask tick by tick (S * A * L < 2^31,
// checked on the host).
struct ProfileTraceArgs {
    ProfileArgs p;           // f, rows, per_level, cand and L (rank, pair_off, key_of and key are not read)
    const float* level_rpm;  // [L * S] row t's arrival rates ...
    const int* level_in;     // ... input tokens ...
    const int* level_out;    // ... and output tokens
};
__global__ void profile_trace_kernel(ProfileTraceArgs g) {
    const ProfileArgs& p = g.p;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_pairs = p.f.S * p.f.A;
    if (i >= n_pairs * p.L) return;
    const int t = i / n_pairs, pair = i - t * n_pairs;
    const int s = pair / p.f.A, a = pair % p.f.A;
    DevFleet ft = profile_at(p, t);
    ft.srv_arrival_rpm = g.level_rpm + (size_t)t * p.f.S;
    ft.srv_in_tokens = g.level_in + (size_t)t * p.f.S;
    ft.srv_out_tokens = g.level_out + (size_t)t * p.f.S;
    const int cls = pair_class(ft, s, a, true);
    Cand c = cand_nil();
    if (cls == PAIR_ZERO) c = zero_load_alloc(ft, s, a);
    else if (cls == PAIR_LOAD) c = priced_at(ft, ft.srv_model[s], a, load_cand(p.cand, i));
    store_cand(p.cand, i, c);
}

// wva_size_grid's value + per-server minimum: one warp per server over its A * B candidates (record
// (s * A + a) * B + bi), strided, so any A * B fits.  Every feasible candidate gets value = TransitionPenalty as in
// unlimited_kernel.  The winner is SolveUnlimited's (strict '<' from MaxFloat32: a NaN value or one not below
// MaxFloat32 never wins), ties to the smaller batch size, then the lower accelerator id, then the lower bi
// (repeated batch sizes give identical records).
struct SgKey {
    float value;
    int batch, a, bi;  // bi < 0: none
};
__device__ __forceinline__ bool sg_better(const SgKey& x, const SgKey& y) {
    if (x.bi < 0) return false;
    if (y.bi < 0) return true;
    if (x.value != y.value) return x.value < y.value;
    if (x.batch != y.batch) return x.batch < y.batch;
    if (x.a != y.a) return x.a < y.a;
    return x.bi < y.bi;
}
__global__ void __launch_bounds__(128) size_grid_finalize(DevFleet f, AllocCols cand, const int* batch, int B,
                                                          AllocCols winners) {
    const int s = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (s >= f.S) return;
    const int n = f.A * B;
    const size_t base = (size_t)s * n;
    SgKey best{0.0f, 0, 0, -1};
    for (int k = lane; k < n; k += 32) {
        if (!cand.feasible[base + k]) continue;
        const float v = penalty_of(f, s, load_cand(cand, base + k));
        cand.value[base + k] = v;
        const int a = k / B, bi = k - a * B;
        const SgKey key{v, batch[bi], a, bi};
        if (v < 3.40282346638528859811704183484516925440e+38f && sg_better(key, best)) best = key;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        SgKey o;
        o.value = __shfl_down_sync(0xffffffffu, best.value, d);
        o.batch = __shfl_down_sync(0xffffffffu, best.batch, d);
        o.a = __shfl_down_sync(0xffffffffu, best.a, d);
        o.bi = __shfl_down_sync(0xffffffffu, best.bi, d);
        if (sg_better(o, best)) best = o;
    }
    if (lane == 0) {
        Cand c = cand_nil();
        if (best.bi >= 0) {
            c = load_cand(cand, base + (size_t)best.a * B + best.bi);
            c.value = best.value;
        }
        store_cand(winners, s, c);
    }
}

// ---------------------------------------------------------------------------
// What Manager.Optimize / Solver.Solve leave behind next to the solution: System.AllocateByType
// (pkg/core/system.go:271-300) and CreateAllocationDiff per server (pkg/core/allocation.go:353-380,
// pkg/solver/solver.go:51-58).  One CTA: the diffs are element-wise; the per-type totals add float32
// costs in ascending server index (the reference's own order is Go map order), so thread t owns type t
// and walks the servers in order, chunk by chunk through shared memory (coalesced loads, serial adds).
// ---------------------------------------------------------------------------
struct SummaryOut {
    uint8_t* type_present;
    long long* type_count;
    int* type_limit;
    float* type_cost;
    int *diff_old_acc, *diff_new_acc, *diff_old_replicas, *diff_new_replicas;
    float* diff_cost;
};
constexpr int kSumChunk = 1024;
constexpr int kSumMaxTypes = 1024;  // 256 threads x 4 owned types
__global__ void __launch_bounds__(256) summary_kernel(DevFleet f, AllocCols win, SummaryOut o) {
    __shared__ int s_type[kSumChunk];
    __shared__ long long s_units[kSumChunk];
    __shared__ float s_cost[kSumChunk];
    // one accumulator set per owned type (thread t owns types t, t + 256, ...: at most 4 in registers)
    constexpr int kOwn = 4;
    long long cnt[kOwn];
    float cost[kOwn];
    int present[kOwn];
#pragma unroll
    for (int k = 0; k < kOwn; ++k) { cnt[k] = 0; cost[k] = 0.0f; present[k] = 0; }
    for (int base = 0; base < f.S; base += kSumChunk) {
        const int n = min(kSumChunk, f.S - base);
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int s = base + i;
            const int feas = win.feasible[s], acc = win.acc[s], rep = win.replicas[s];
            const float c = win.cost[s];
            int type = -1;
            long long units = 0;
            const int m = f.srv_model[s];
            if (feas && acc >= 0 && acc < f.A && m >= 0 && m < f.M) {  // system.go:276-284
                const int t = f.acc_type[acc];
                if (t >= 0 && t < f.T) {
                    type = t;
                    const long long inst = f.perf_present[m * f.A + acc] ? num_instances(f, m, acc) : 0;
                    units = (long long)rep * inst * (long long)f.acc_mult[acc];  // :296
                }
            }
            s_type[i] = type;
            s_units[i] = units;
            s_cost[i] = c;
            // CreateAllocationDiff(current, solution)
            if (o.diff_old_acc) o.diff_old_acc[s] = f.srv_cur_acc[s];
            if (o.diff_old_replicas) o.diff_old_replicas[s] = f.srv_cur_replicas[s];
            if (o.diff_new_acc) o.diff_new_acc[s] = feas ? acc : -3;
            if (o.diff_new_replicas) o.diff_new_replicas[s] = feas ? rep : 0;
            if (o.diff_cost) o.diff_cost[s] = __fsub_rn(feas ? c : 0.0f, f.srv_cur_cost[s]);
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kOwn; ++k) {
            const int t = threadIdx.x + k * blockDim.x;
            if (t < f.T) {
                for (int i = 0; i < n; ++i)
                    if (s_type[i] == t) {
                        present[k] = 1;
                        cnt[k] += s_units[i];
                        cost[k] = __fadd_rn(cost[k], s_cost[i]);  // :297, float32
                    }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < kOwn; ++k) {
        const int t = threadIdx.x + k * blockDim.x;
        if (t < f.T) {
            if (o.type_present) o.type_present[t] = (uint8_t)present[k];
            if (o.type_count) o.type_count[t] = cnt[k];
            if (o.type_limit) o.type_limit[t] = f.type_capacity[t];
            if (o.type_cost) o.type_cost[t] = cost[k];
        }
    }
}

// ---------------------------------------------------------------------------
// MM1KModel (closed form): pkg/analyzer/mm1kmodel.go:19-92 over QueueModel.Solve (queuemodel.go:27-37).  One
// thread per (K, lambda, mu) triple; the probabilities are streamed in the reference's order (sumP and the
// sum(i p[i]) accumulate over i = 0..K), never stored.
// ---------------------------------------------------------------------------
struct Mm1kArgs {
    int n;
    const int* K;
    const float* lambda;
    const float* mu;
    uint8_t* is_valid;
    float *rho, *avg_num_in_system, *throughput, *avg_resp_time, *avg_serv_time, *avg_wait_time, *avg_queue_length;
    double* sum_p;
};
__global__ void __launch_bounds__(128) mm1k_kernel(Mm1kArgs g) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= g.n) return;
    const int K = g.K[q];
    const float lambda = g.lambda[q], mu = g.mu[q];
    const float rho = (lambda == mu) ? 1.0f : __fdiv_rn(lambda, mu);  // ComputeRho: mm1kmodel.go:38-44
    // QueueModel.Solve validity: queuemodel.go:31 with GetRhoMax = K (mm1kmodel.go:46-48)
    const bool valid = !((rho < 0.0f) || (rho >= (float)K) || (lambda < 0.0f) || (mu <= 0.0f));
    float nsys = 0.f, thr = 0.f, resp = 0.f, serv = 0.f, wait = 0.f, qlen = 0.f;
    double sum_p = 0.0;
    if (valid) {
        const double r = (double)rho;
        // computeProbabilities: mm1kmodel.go:51-72
        const double p0 = (rho == 1.0f) ? __ddiv_rn(1.0, (double)(K + 1))
                                        : __ddiv_rn(__dsub_rn(1.0, r), __dsub_rn(1.0, go_pow_uint(r, (long long)K + 1)));
        double temp = 0.0, pK = 0.0;
        for (int i = 0; i <= K; ++i) {
            const double pi = __dmul_rn(p0, go_pow_uint(r, (long long)i));
            sum_p = __dadd_rn(sum_p, pi);
            temp = __dadd_rn(temp, __dmul_rn((double)i, pi));  // computeStatistics: :75-92
            pK = pi;
        }
        nsys = (float)temp;
        thr = __fmul_rn(lambda, __fsub_rn(1.0f, (float)pK));
        resp = __fdiv_rn(nsys, thr);
        serv = __fdiv_rn(1.0f, mu);
        wait = __fsub_rn(resp, serv);
        if (wait < 0.0f) wait = 0.0f;
        qlen = __fmul_rn(thr, wait);
    }
    g.is_valid[q] = valid ? 1 : 0;
    g.rho[q] = rho;
    g.avg_num_in_system[q] = nsys;
    g.throughput[q] = thr;
    g.avg_resp_time[q] = resp;
    g.avg_serv_time[q] = serv;
    g.avg_wait_time[q] = wait;
    g.avg_queue_length[q] = qlen;
    g.sum_p[q] = sum_p;
}

// ---------------------------------------------------------------------------
// Latency sweep: warp = 32 consecutive rates of one (server, acc) pair.
// ---------------------------------------------------------------------------
struct SweepArgs {
    DevFleet f;
    const int* pair_list;  // pairs sorted by descending N
    const int* pair_N;     // N per entry of pair_list
    const long long* tab_off;  // shared-table entry offset per entry of pair_list
    const double* tab;
    int n_pairs, n_rates, n_chunks;
    unsigned* counter;
    uint8_t* valid;
    float *rate, *ttft, *itl, *throughput, *rho;
    FbList fb;             // points that bailed: fb_pack(entry of pair_list, rate index)
};

// The sweep's rate i of a pair (same float32 expressions as the oracle's sweep).
__device__ __forceinline__ float sweep_rate(float rmin, float rmax, int i, int n_rates) {
    const float hi = __fmul_rn(rmax, 0.999f);
    const float span = __fsub_rn(hi, rmin);
    const float frac = n_rates > 1 ? __fdiv_rn((float)i, (float)(n_rates - 1)) : 0.0f;
    return __fadd_rn(rmin, __fmul_rn(span, frac));
}

__global__ void __launch_bounds__(256) sweep_kernel(SweepArgs g) {
    const DevFleet& f = g.f;
    const int lane = threadIdx.x & 31;
    const unsigned n_items = (unsigned)g.n_pairs * g.n_chunks;
    for (;;) {
        unsigned item = 0;
        if (lane == 0) item = atomicAdd(g.counter, 1u);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= n_items) break;
        const int e = item / g.n_chunks, chunk = item % g.n_chunks;
        const int pair = g.pair_list[e];
        const int s = pair / f.A, a = pair % f.A;
        const int N = g.pair_N[e], K = N + N * f.ratio;
        const double* tab = g.tab + 4 * g.tab_off[e];
        Recip tail;
        tail.b = tab[4 * (N - 1)];
        tail.yh = tab[4 * (N - 1) + 1];
        tail.yl = tab[4 * (N - 1) + 2];
        const float rmin = rate_min_of((float)tab[0]), rmax = rate_max_of((float)tail.b);
        const int i = chunk * 32 + lane;
        if (i < g.n_rates) {
        const float rate = sweep_rate(rmin, rmax, i, g.n_rates);
        const size_t o = (size_t)pair * g.n_rates + i;
        g.rate[o] = rate;
        uint8_t ok = 0;
        Metrics m;
        m.ttft = m.avg_token_time = m.rho = m.throughput = 0.0f;
        if (!(rate <= 0.0f) && !(rate > rmax) && K >= 2) {
            ModelStats st;
            const QParams q = qparams_of(f, s, a);
            if (solve_shared(tab, N, K, __fdiv_rn(rate, 1000.0f), st) == kSolveOk) {
                m = metrics_from(q, N, st);
                ok = 1;
            } else {
                fb_push(g.fb, fb_pack(e, i));
            }
        }
        g.valid[o] = ok;
        g.ttft[o] = m.ttft;
        g.itl[o] = m.avg_token_time;
        g.throughput[o] = m.throughput;
        g.rho[o] = m.rho;
        }
    }
}

// Stored-vector re-run of the sweep points sweep_kernel bailed on.
__global__ void sweep_fallback(SweepArgs g, FbRun r) {
    const DevFleet& f = g.f;
    fb_rerun(r, [&](unsigned long long item, double* p) {
        const int e = (int)(item >> 32), i = (int)(unsigned)item;
        const int pair = g.pair_list[e];
        const int s = pair / f.A, a = pair % f.A;
        const int N = g.pair_N[e], K = N + N * f.ratio;
        const double* tab = g.tab + 4 * g.tab_off[e];
        const float rate = sweep_rate(rate_min_of((float)tab[0]), rate_max_of((float)tab[4 * (N - 1)]), i, g.n_rates);
        ModelStats st;
        const int rc = solve_stored(p, tab, N, K, __fdiv_rn(rate, 1000.0f), st);
        if (rc != 0) return rc;
        const Metrics m = metrics_from(qparams_of(f, s, a), N, st);
        const size_t o = (size_t)pair * g.n_rates + i;
        g.valid[o] = 1;
        g.ttft[o] = m.ttft;
        g.itl[o] = m.avg_token_time;
        g.throughput[o] = m.throughput;
        g.rho[o] = m.rho;
        return 0;
    });
}

}  // namespace wva

// wva_size.cuh — K1, the reference's decision path: CreateAllocation (pkg/core/allocation.go:27-163) for every
// (server, accelerator) candidate.  The decisions (the start, the bisections' end-point test and walk, lambda*, the
// replica count, the feasible candidate) are written once below and driven two ways: large fleets run ROUNDS of
// sorted solve batches with SPECULATIVE bisection (sz2_*); small fleets and the stored-vector fallback run
// create_allocation straight through (size_warp_kernel, size_fallback).  The load grid runs the same drivers up to
// rateStar (the part that does not read the load), then its tail per load level (load_kernel, load_fallback); the
// workload grid runs them on a fleet of token keys, then the same tail (workload_kernel, workload_fallback).
//
// The reference runs, per candidate, two sequential bisections (pkg/analyzer/utils.go:26-70) of <= 102 model
// solves each, then two Analyze calls.  The solves of one bisection depend on each other only through ONE
// comparison per iteration, and the next midpoint can only be one of two values; so a round evaluates the whole
// binary tree of midpoints the next D iterations can reach (2^D - 1 solves: node 1 = mid(lo, hi), node 2v / 2v + 1 =
// the midpoints after "target below" / "target above" at node v), and the state machine then walks the tree with
// the reference's comparisons, tolerance test and iteration count.  Every lambda is produced by the reference's own
// float32 expression 0.5 * (xmin + xmax) on the reference's own bounds, so the D iterations a round resolves are
// the reference's iterations, bit for bit; the evaluations off the taken path are discarded.  D iterations per
// round instead of one: ~36 rounds become ~36 / D + 3.
//
// Why this is also the fix for the memory traffic: every candidate owns a service-rate table (its token profile is
// its own), and with one request per candidate per round each lane of a solve warp streamed a different table
// (hundreds of MB of DRAM reads per round on 100 k candidates).  The 2 x (2^D - 1) requests of a
// candidate share ONE table; they are emitted into consecutive slots and, once the interval has narrowed, fall
// into the same length class, so the sort keeps them adjacent and a solve warp reads a few tables instead of 32.
//
// Rounds are enqueued without host synchronisation (grids sized for the worst case, every kernel leaves at once
// when its work list is empty); the host looks at the request counter once per group of rounds.
#pragma once
#include "wva_kernels.cuh"

namespace wva {

constexpr int kSzMaxDepth = 5;  // midpoint tree depth: at most 31 evaluations per search per round

// Where a candidate's table and record are.  wva_solve: one table per candidate (N entries, table index j) and
// record = pair id.  wva_size_grid: the candidates of one pair at its batch sizes share the pair's table of Bmax
// >= N entries and write record pair * B + bi.  A longer table changes no result: the solves read entries 0..N-1,
// and column 4's suffix minimum at n is then min(servRate[n..Bmax-1]), a lower bound of the minimum over the
// rates the chain reads (servRate[n..N-1]), so the early exit (rate_below) fires only where it would have fired on
// an N-long table, and the exponent bound from entry 0's suffix minimum only narrows the block windows
// (grid_kernel's cells rely on the same).
struct CandPlace {
    const int* tab_idx;   // [n_cand] table index, for the ls column (NULL: j)
    const int* rec;       // [n_cand] output record (NULL: the pair id)
    __device__ __forceinline__ int record(int j, int pair) const { return rec ? rec[j] : pair; }
    __device__ __forceinline__ const float* ls_of(const float* ls, const long long* tab_off, int j) const {
        return ls + tab_off[j] + (tab_idx ? tab_idx[j] : j);  // a table of len entries has len + 1 ls entries
    }
};

// Search mode's candidate columns (the SLO grid): the one search a candidate runs, and its target.
struct SearchCols {
    const uint8_t* which;  // [n_cand] 0: TTFT, 1: ITL
    const float* target;   // [n_cand] the target, > 0
};

struct SizeArgs {
    DevFleet f;
    const int* cand_pair;      // [n_cand] pair ids sorted by descending N
    const int* cand_N;         // [n_cand]
    int n_cand;
    const double* tab;         // shared-format tables
    const long long* tab_off;  // [n_cand] entry offset of the candidate's table
    const float* ls;           // prefix log2 sums of the tables (scheduling estimate only)
    CandPlace place;
    AllocCols cand;
    FbList fb;                 // candidate indices that bailed
};
// ... with search mode's columns (size_warp_search, size_fallback_search)
struct SearchArgs {
    SizeArgs g;
    SearchCols search;
};

// The rounds' sort workspace and its item ordering kernels.
struct SortWs {
    unsigned* order;
    unsigned long long* items;
    unsigned long long* items_sorted;
    unsigned* item_count;  // [0] items, [1..256] per class, [257..512] cursors
};
__global__ void __launch_bounds__(256) ws_items_scan(SortWs ws) {
    __shared__ unsigned tot[kClasses];
    tot[threadIdx.x] = ws.item_count[1 + threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned acc = 0;
        for (int c = 0; c < kClasses; ++c) {
            ws.item_count[1 + kClasses + c] = acc;
            acc += tot[c];
        }
    }
}
__global__ void __launch_bounds__(256) ws_items_scatter(SortWs ws) {
    const unsigned n = *ws.item_count;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long it = ws.items[i];
    ws.items_sorted[agg_inc(ws.item_count + 1 + kClasses, (int)((it >> 40) & 0xff))] = it;
}

// candidate phase (rounds)
enum { PH_SEARCH = 0, PH_WAIT_STAR = 1, PH_WAIT_FINAL = 2, PH_DONE = 3, PH_NIL = 4, PH_BAIL = 5 };

enum { SZ2_START = 0, SZ2_WAIT_FIRST = 1, SZ2_WAIT_ITER = 2, SZ2_DONE = 3, SZ2_OFF = 4 };

struct Sz2Args {
    DevFleet f;
    const int* cand_pair;  // [n] pair ids, descending N
    const int* cand_N;     // [n]
    int n_cand;
    int depth;             // D
    const double* tab;     // shared-format tables
    const long long* tab_off;  // [n]
    const float* ls;
    CandPlace place;
    // search state, index 2*j + which (0: TTFT, 1: ITL)
    float *xmin, *xmax, *xs;
    uint8_t *sst, *inc, *iter;
    int8_t* ind;
    int* slot;             // [2n] first request slot of the search this round
    // candidate state
    uint8_t* phase;
    float *rmax, *l2s0, *l2sN, *lsN, *rate_star, *cost;
    long long* nrep;
    int* aslot;            // [n] request slot of the candidate's Analyze this round
    // requests of the current round
    unsigned* req_id;      // 4*j + kind (0 TTFT eval, 1 ITL eval, 2 Analyze(lambda*), 3 Analyze(final))
    float* req_lam;
    uint8_t* req_key;
    float4* req_out;       // kinds 0/1: x = y; kinds 2/3: throughput, ttft, itl, rho
    uint8_t* req_bail;
    unsigned* n_req;       // device counter of this round
    unsigned* n_live;      // device counter: candidates that are not finished yet (host stop test)
    SortWs ws;
    AllocCols cand;
    FbList fb;
    SearchCols search;     // search mode only
};

// ---------------------------------------------------------------------------
// The decision pieces of CreateAllocation, shared by every driver.  They do not know where an evaluation ran: a
// driver hands them {y, bail} per evaluated point, and a bail-out of a point they never consult is ignored.
// ---------------------------------------------------------------------------
struct SzPt {
    float y;
    bool bail;
};
enum { SZ_MORE = 0, SZ_DONE = 1, SZ_BAIL = 2 };

__device__ __forceinline__ float sz_mid(float lo, float hi) { return __fmul_rn(0.5f, __fadd_rn(lo, hi)); }  // utils.go:55

// Midpoint of heap node v (1-based) of the tree over (lo, hi): follow v's path bits below its leading one.
__device__ __forceinline__ float sz_node_value(int v, float lo, float hi) {
    const int depth = 31 - __clz(v);
    for (int b = depth - 1; b >= 0; --b) {
        const float x = sz_mid(lo, hi);
        if ((v >> b) & 1) lo = x; else hi = x;
    }
    return sz_mid(lo, hi);
}

// EvalTTFT (which = 0) / EvalITL (which = 1) from the solved model: queueanalyzer.go:270-290.
__device__ __forceinline__ float target_value(const QParams& q, int which, int N, const ModelStats& st) {
    const float eff = effective_concurrency(q, st.avg_serv_time, N);
    return which == 0 ? __fadd_rn(st.avg_wait_time, prefill_time(q, eff)) : decode_time(q, eff);
}

// The start of CreateAllocation: RateRange and the bisection bounds.  nil: a model with K <= 1 is never valid
// (queuemodel.go:31), negative targets fail TargetPerf.check (:322-329), and a bisection with lambda_min >
// lambda_max returns an error before it evaluates anything (utils.go:29-31).
struct SzStart {
    float rmax, lmin, lmax;
    bool nil;
};
// RateRange in req/s and the bisection bounds lambda_min / lambda_max in req/ms (queueanalyzer.go:197-198) from a
// table's first and last service rates.
__device__ __forceinline__ void sz_range(float s1, float sN, float& rmax, float& lmin, float& lmax) {
    rmax = rate_max_of(sN);
    lmin = __fdiv_rn(rate_min_of(s1), 1000.0f);
    lmax = __fdiv_rn(rmax, 1000.0f);
}
__device__ __forceinline__ SzStart sz_start(const DevFleet& f, int s, int K, float s1, float sN) {
    SzStart b;
    sz_range(s1, sN, b.rmax, b.lmin, b.lmax);
    const float slo_ttft = f.srv_slo_ttft[s], slo_itl = f.srv_slo_itl[s], slo_tps = f.srv_slo_tps[s];
    b.nil = K < 2 || slo_itl < 0.0f || slo_ttft < 0.0f || slo_tps < 0.0f ||
            (b.lmin > b.lmax && (slo_ttft > 0.0f || slo_itl > 0.0f));
    return b;
}

// One BinarySearch (utils.go:26-70).  xs = lambdaStar so far; ind < 0: "target is below the bounded region".
struct SzSearch {
    float lo, hi, xs;
    int it, ind;
    bool inc;
};

// The two boundary evaluations (utils.go:36-51); end(0) / end(1) = the points at lo / hi.  A bail-out at hi
// counts only when the point at lo was not within tolerance.  The SLO bounds class their targets with it too.
template <class End>
__device__ __forceinline__ int sz_ends(SzSearch& S, float target, End&& end) {
    const SzPt p0 = end(0);
    if (p0.bail) return SZ_BAIL;
    if (within_tolerance(p0.y, target, 1e-6f)) { S.xs = S.lo; return SZ_DONE; }
    const SzPt p1 = end(1);
    if (p1.bail) return SZ_BAIL;
    if (within_tolerance(p1.y, target, 1e-6f)) { S.xs = S.hi; return SZ_DONE; }
    const float y0 = p0.y, y1 = p1.y;
    S.inc = y0 < y1;
    if ((S.inc && target < y0) || (!S.inc && target > y0)) { S.xs = S.lo; S.ind = -1; return SZ_DONE; }
    if ((S.inc && target > y1) || (!S.inc && target < y1)) { S.xs = S.hi; S.ind = 1; return SZ_DONE; }
    return SZ_MORE;
}

// Up to D iterations of the bisection (utils.go:54-68) over a tree of evaluated midpoints: node(v) is the point
// of heap node v over the current (lo, hi) (sz_node_value).
template <class Node>
__device__ __forceinline__ int sz_walk(SzSearch& S, float target, int D, Node&& node) {
    int v = 1;
    for (int level = 0; level < D; ++level) {
        const SzPt p = node(v);
        if (p.bail) return SZ_BAIL;
        S.xs = sz_mid(S.lo, S.hi);
        if (within_tolerance(p.y, target, 1e-6f)) return SZ_DONE;
        const float pmin = S.lo, pmax = S.hi;
        if ((S.inc && target < p.y) || (!S.inc && target > p.y)) { S.hi = S.xs; v = 2 * v; }
        else { S.lo = S.xs; v = 2 * v + 1; }
        ++S.it;
        // fixed point of the float32 interval: the remaining iterations repeat this solve
        if ((S.lo == pmin && S.hi == pmax) || S.it >= 100) return SZ_DONE;
    }
    return SZ_MORE;
}

// Analyze's rate check (queueanalyzer.go:135-143): false when it rejects the rate, else the lambda it solves at.
__device__ __forceinline__ bool sz_gate(float rate, float rmax, float& lam) {
    if (rate <= 0.0f || rate > rmax) return false;
    lam = __fdiv_rn(rate, 1000.0f);
    return true;
}

// queueanalyzer.go:231-241: lambda = min(lambdaStarTTFT, lambdaStarITL, lambdaStarTPS), then Analyze's check.
__device__ __forceinline__ bool sz_lambda(const DevFleet& f, int s, float rmax, float xs_ttft, float xs_itl,
                                          float& lam) {
    const float lmax = __fdiv_rn(rmax, 1000.0f);
    float l_tps = lmax;
    if (f.srv_slo_tps[s] > 0.0f) l_tps = __fmul_rn(lmax, __fsub_rn(1.0f, 0.1f));
    return sz_gate(__fmul_rn(go_minf(go_minf(xs_ttft, xs_itl), l_tps), 1000.0f), rmax, lam);
}

// allocation.go:140-153: replicas and cost for the throughput rate_star at totalRate (:134-139, total_rate_of),
// then Analyze's check of the final rate.
struct SzReplicas {
    long long nrep;
    float cost;
};
// ceil(totalRate / rateStar) before the conversion to int (allocation.go:141)
__device__ __forceinline__ double sz_quotient(float total_rate, float rate_star) {
    return ceil(__ddiv_rn((double)total_rate, (double)rate_star));
}
// the per-replica rate Analyze checks (allocation.go:146)
__device__ __forceinline__ float sz_final_rate(float total_rate, long long nrep) {
    return __fdiv_rn(total_rate, (float)nrep);
}
__device__ __forceinline__ bool sz_replicas(const DevFleet& f, int s, int a, float rmax, float rate_star,
                                            float total_rate, SzReplicas& r, float& lam) {
    r.nrep = go_f64_to_int(sz_quotient(total_rate, rate_star));
    const long long min_rep = f.srv_min_replicas[s];
    if (r.nrep < min_rep) r.nrep = min_rep;
    const long long total = (long long)num_instances(f, f.srv_model[s], a) * r.nrep;
    r.cost = __fmul_rn(f.acc_cost[a], (float)total);
    return sz_gate(sz_final_rate(total_rate, r.nrep), rmax, lam);
}

// The feasible allocation (allocation.go:155-163); value = cost.
__device__ __forceinline__ Cand sz_cand(int a, int N, const SzReplicas& r, float rate_star, float ttft, float itl,
                                        float rho) {
    Cand c = cand_nil();
    c.feasible = 1;
    c.acc = a;
    c.replicas = (int)r.nrep;
    c.batch = N;
    c.cost = r.cost;
    c.value = r.cost;
    c.itl = itl;
    c.ttft = ttft;
    c.rho = rho;
    c.max_rate = __fdiv_rn(rate_star, 1000.0f);
    return c;
}

// rateStar mode's record of a candidate whose sizing succeeded: feasible, max_rate = rateStar (req/s, not yet
// divided by 1000).  The caller passes only the feasible and max_rate columns.
__device__ __forceinline__ Cand star_cand(float rate_star) {
    Cand c = cand_nil();
    c.feasible = 1;
    c.max_rate = rate_star;
    return c;
}

// Search mode's record of one search, in the feasible and max_rate columns: SEARCH_NIL (K < 2, lambda_min >
// lambda_max, or "target is below the bounded region"), SEARCH_OK with max_rate = lambdaStar (req/ms), or
// SEARCH_FAIL: a solve's rescale loop does not terminate (the stored-vector re-run failed).  The search fallback
// does not raise the call's status for SEARCH_FAIL: only a caller whose reference would have run the search does.
enum { SEARCH_NIL = 0, SEARCH_OK = 1, SEARCH_FAIL = 2 };
__device__ __forceinline__ Cand search_cand(int status, float xs) {
    Cand c = cand_nil();
    c.feasible = (uint8_t)status;
    c.max_rate = xs;
    return c;
}
// The search's target: search mode's column, else the server's own (which = 0: TTFT, 1: ITL).
template <bool kSearch>
__device__ __forceinline__ float search_target(const DevFleet& f, const SearchCols& sc, int j, int s, int which) {
    if constexpr (kSearch) return which == sc.which[j] ? sc.target[j] : 0.0f;
    return which == 0 ? f.srv_slo_ttft[s] : f.srv_slo_itl[s];
}

// ---------------------------------------------------------------------------
// The rounds (more than WVA_SIZE_SMALL_MAX candidates): one thread per candidate keeps the search state in global
// columns between rounds; both searches of a candidate emit their trees in the same round.
// ---------------------------------------------------------------------------
// kSearch: search mode (the SLO grid), where a candidate runs only its one search and is nil only for K < 2 or an
// empty range.
template <bool kSearch>
__device__ __forceinline__ void sz2_init_body(const Sz2Args& g) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= g.n_cand) return;
    const DevFleet& f = g.f;
    const int pair = g.cand_pair[j], s = pair / f.A;
    const int N = g.cand_N[j], K = N + N * f.ratio;
    const double* tab = g.tab + 4 * g.tab_off[j];
    const float s1 = (float)tab[0], sN = (float)tab[4 * (N - 1)];
    SzStart b = sz_start(f, s, K, s1, sN);
    if constexpr (kSearch) b.nil = K < 2 || b.lmin > b.lmax;
    g.rmax[j] = b.rmax;
    g.l2s0[j] = log2f(s1);
    g.l2sN[j] = log2f(sN);
    g.lsN[j] = g.place.ls_of(g.ls, g.tab_off, j)[N - 1];
    g.phase[j] = b.nil ? PH_NIL : PH_SEARCH;
    for (int w = 0; w < 2; ++w) {
        const float target = search_target<kSearch>(f, g.search, j, s, w);
        g.xmin[2 * j + w] = b.lmin;
        g.xmax[2 * j + w] = b.lmax;
        g.xs[2 * j + w] = b.lmax;  // lambdaStar when the target is disabled (queueanalyzer.go:205,218)
        g.sst[2 * j + w] = target > 0.0f ? SZ2_START : SZ2_OFF;
        g.ind[2 * j + w] = 0;
        g.inc[2 * j + w] = 0;
        g.iter[2 * j + w] = 0;
        g.slot[2 * j + w] = -1;
    }
    g.aslot[j] = -1;
    if (b.nil) store_cand(g.cand, g.place.record(j, pair), cand_nil());
}
__global__ void __launch_bounds__(256) sz2_init(Sz2Args g) { sz2_init_body<false>(g); }
__global__ void __launch_bounds__(256) sz2_init_search(Sz2Args g) { sz2_init_body<true>(g); }

// Advance every candidate: consume last round's results (walking the midpoint trees with the reference's
// comparisons), then emit this round's requests into consecutive slots.  kStar: rateStar mode, kSearch: search
// mode (create_allocation).
template <bool kStar, bool kSearch = false>
__device__ __forceinline__ void sz2_advance_body(const Sz2Args& g) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const DevFleet& f = g.f;
    const int D = g.depth, M = (1 << D) - 1;
    const int lane = threadIdx.x & 31;
    int ph = PH_DONE;
    int pair = 0, s = 0, a = 0;
    float rmax = 0.0f;
    if (j < g.n_cand) {
        ph = g.phase[j];
        pair = g.cand_pair[j];
        s = pair / f.A;
        a = pair % f.A;
        rmax = g.rmax[j];
    }
    const bool live_in = ph < PH_DONE;
    // what this thread will emit: per search a tree (optionally preceded by the two end points), or one Analyze
    int emit_n[2] = {0, 0};
    bool emit_ends[2] = {false, false};
    float emit_lo[2] = {0.f, 0.f}, emit_hi[2] = {0.f, 0.f};
    int an_kind = -1;
    float an_lambda = 0.0f;
    if (live_in) {
        if (ph == PH_SEARCH) {
            bool all_done = true, nil = false, bail = false;
            for (int w = 0; w < 2; ++w) {
                const int k = 2 * j + w;
                int st = g.sst[k];
                if (st == SZ2_DONE || st == SZ2_OFF) continue;
                const float target = search_target<kSearch>(f, g.search, j, s, w);
                float lo = g.xmin[k], hi = g.xmax[k];
                if (st == SZ2_START) {
                    emit_ends[w] = true;
                    st = SZ2_WAIT_FIRST;
                } else {  // last round's points: the two end points (first round only), then the tree
                    SzSearch S{lo, hi, g.xs[k], g.iter[k], g.ind[k], g.inc[k] != 0};
                    const int base = g.slot[k];
                    auto at = [&](int i) { return SzPt{g.req_out[base + i].x, g.req_bail[base + i] != 0}; };
                    int r = SZ_MORE;
                    const int nodes = st == SZ2_WAIT_FIRST ? 2 : 0;
                    if (st == SZ2_WAIT_FIRST) r = sz_ends(S, target, at);
                    if (r == SZ_MORE) r = sz_walk(S, target, D, [&](int v) { return at(nodes + v - 1); });
                    if (r == SZ_BAIL) { bail = true; break; }
                    if (r == SZ_DONE && S.ind < 0) { nil = true; break; }  // "target is below the bounded region"
                    g.xmin[k] = lo = S.lo;
                    g.xmax[k] = hi = S.hi;
                    g.xs[k] = S.xs;
                    g.iter[k] = (uint8_t)S.it;
                    g.ind[k] = (int8_t)S.ind;
                    g.inc[k] = S.inc;
                    st = r == SZ_DONE ? SZ2_DONE : SZ2_WAIT_ITER;
                }
                g.sst[k] = (uint8_t)st;
                if (st != SZ2_DONE) {
                    emit_n[w] = M + (emit_ends[w] ? 2 : 0);
                    emit_lo[w] = lo;
                    emit_hi[w] = hi;
                    all_done = false;
                }
            }
            if (bail) ph = PH_BAIL;
            else if (nil) ph = PH_NIL;
            else if (kSearch && all_done) {
                store_cand(g.cand, g.place.record(j, pair), search_cand(SEARCH_OK, g.xs[2 * j + g.search.which[j]]));
                ph = PH_DONE;
            } else if (all_done) {
                if (!sz_lambda(f, s, rmax, g.xs[2 * j], g.xs[2 * j + 1], an_lambda)) ph = PH_NIL;
                else { an_kind = 2; ph = PH_WAIT_STAR; }
            }
            if (ph != PH_SEARCH) emit_n[0] = emit_n[1] = 0;
        } else if (ph == PH_WAIT_STAR) {
            const int slot = g.aslot[j];
            if (g.req_bail[slot]) ph = PH_BAIL;
            else {
                const float rate_star = g.req_out[slot].x;  // metrics.Throughput
                if constexpr (kStar) {
                    store_cand(g.cand, g.place.record(j, pair), star_cand(rate_star));
                    ph = PH_DONE;
                } else {
                    SzReplicas r;
                    const bool ok = sz_replicas(f, s, a, rmax, rate_star, total_rate_of(f, s), r, an_lambda);
                    g.rate_star[j] = rate_star;
                    g.nrep[j] = r.nrep;
                    g.cost[j] = r.cost;
                    if (!ok) ph = PH_NIL;
                    else { an_kind = 3; ph = PH_WAIT_FINAL; }
                }
            }
        } else {  // PH_WAIT_FINAL
            const int slot = g.aslot[j];
            if (g.req_bail[slot]) ph = PH_BAIL;
            else {
                const float4 m = g.req_out[slot];
                const SzReplicas r{g.nrep[j], g.cost[j]};
                store_cand(g.cand, g.place.record(j, pair), sz_cand(a, g.cand_N[j], r, g.rate_star[j], m.y, m.z, m.w));
                ph = PH_DONE;
            }
        }
        if (ph == PH_NIL) store_cand(g.cand, g.place.record(j, pair), cand_nil());
        if (ph == PH_BAIL) {
            fb_push(g.fb, (unsigned)j);
            store_cand(g.cand, g.place.record(j, pair), cand_nil());
        }
        g.phase[j] = (uint8_t)ph;
    }
    // ---- consecutive request slots per thread: warp scan of the counts, one atomic per warp ----
    const int mine = emit_n[0] + emit_n[1] + (an_kind >= 0 ? 1 : 0);
    int incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    const int warp_total = __shfl_sync(0xffffffffu, incl, 31);
    unsigned warp_base = 0;
    if (lane == 31 && warp_total > 0) warp_base = atomicAdd(g.n_req, (unsigned)warp_total);
    warp_base = __shfl_sync(0xffffffffu, warp_base, 31);
    const unsigned live_now = __ballot_sync(0xffffffffu, ph < PH_DONE);
    if (lane == 0 && live_now) atomicAdd(g.n_live, (unsigned)__popc(live_now));
    if (mine == 0) return;
    unsigned slot = warp_base + (unsigned)(incl - mine);
    const int N = g.cand_N[j], K = N + N * f.ratio;
    const long long off = g.tab_off[j];
    const float* ls = g.place.ls_of(g.ls, g.tab_off, j);
    const float l2s0 = g.l2s0[j], l2sN = g.l2sN[j], lsN = g.lsN[j];
    auto put = [&](int kind, float lambda) {
        g.req_id[slot] = (unsigned)j * 4u + (unsigned)kind;
        g.req_lam[slot] = lambda;
        g.req_key[slot] = (uint8_t)length_class(estimate_len(g.tab + 4 * off, ls, N, K, lambda, log2f(lambda),
                                                             l2s0, l2sN, lsN));
        ++slot;
    };
    for (int w = 0; w < 2; ++w) {
        if (emit_n[w] == 0) continue;
        g.slot[2 * j + w] = (int)slot;
        if (emit_ends[w]) {
            put(w, emit_lo[w]);
            put(w, emit_hi[w]);
        }
        for (int v = 1; v <= M; ++v) put(w, sz_node_value(v, emit_lo[w], emit_hi[w]));
    }
    if (an_kind >= 0) {
        g.aslot[j] = (int)slot;
        put(an_kind, an_lambda);
    }
}
__global__ void __launch_bounds__(256) sz2_advance(Sz2Args g) { sz2_advance_body<false>(g); }
__global__ void __launch_bounds__(256) sz2_advance_star(Sz2Args g) { sz2_advance_body<true>(g); }
__global__ void __launch_bounds__(256) sz2_advance_search(Sz2Args g) { sz2_advance_body<false, true>(g); }

// Local counting sort of this round's requests by length class (keys precomputed by sz2_advance); stable inside a
// warp's 32 requests, so the requests of one candidate (consecutive slots) stay adjacent within their class.
__global__ void __launch_bounds__(kSortThreads) sz2_sort_local(Sz2Args g) {
    __shared__ uint8_t keys[kSortChunk];
    __shared__ uint8_t sorted_keys[kSortChunk];
    __shared__ unsigned hist[kClasses];
    __shared__ unsigned cursor[kClasses];
    __shared__ unsigned item_base;
    const unsigned n_req = *g.n_req;
    const unsigned base = blockIdx.x * kSortChunk;
    if (base >= n_req) return;
    if (threadIdx.x < kClasses) hist[threadIdx.x] = 0;
    __syncthreads();
    const int n_here = (int)min((unsigned)kSortChunk, n_req - base);
    for (int k = threadIdx.x; k < n_here; k += kSortThreads) {
        const int key = g.req_key[base + k];
        keys[k] = (uint8_t)key;
        agg_inc(hist, key);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
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
    // one warp pass at a time in request order (warp w takes requests 32 w .. 32 w + 31 of each stripe): a
    // candidate's requests keep their relative order inside a class
    for (int k0 = 0; k0 < n_here; k0 += kSortThreads) {
        const int k = k0 + threadIdx.x;
        if (k < n_here) {
            const int key = keys[k];
            const unsigned pos = agg_inc(cursor, key);
            g.ws.order[base + pos] = base + k;
            sorted_keys[pos] = (uint8_t)key;
        }
    }
    const int n_items = (n_here + 31) >> 5;
    if (threadIdx.x == 0) item_base = atomicAdd(g.ws.item_count, (unsigned)n_items);
    __syncthreads();
    for (int w = threadIdx.x; w < n_items; w += kSortThreads) {
        const unsigned cnt = (unsigned)min(32, n_here - 32 * w);
        const int cls = sorted_keys[32 * w];
        g.ws.items[item_base + w] = (unsigned long long)(base + 32 * w) | ((unsigned long long)cnt << 32) |
                                    ((unsigned long long)cls << 40);
        agg_inc(g.ws.item_count + 1, cls);
    }
}

// One request per lane, 32 requests of similar chain length per warp.
__global__ void __launch_bounds__(256, 4) sz2_solve(Sz2Args g) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned w = idx >> 5, lane = idx & 31;
    if (w >= *g.ws.item_count) return;
    const unsigned long long item = g.ws.items_sorted[w];
    if (lane >= (unsigned)((item >> 32) & 0xff)) return;
    const unsigned slot = g.ws.order[(unsigned)item + lane];
    const unsigned id = g.req_id[slot];
    const int j = (int)(id >> 2), kind = (int)(id & 3);
    const DevFleet& f = g.f;
    const int pair = g.cand_pair[j];
    const int N = g.cand_N[j], K = N + N * f.ratio;
    const float lambda = g.req_lam[slot];
    ModelStats st;
    const int rc = solve_private(g.tab + 4 * g.tab_off[j], N, K, lambda, st);
    g.req_bail[slot] = rc != kSolveOk;
    if (rc != kSolveOk) return;
    const QParams q = qparams_of(f, pair / f.A, pair % f.A);
    float4 out;
    if (kind <= 1) {  // EvalTTFT / EvalITL
        out.x = target_value(q, kind, N, st);
        out.y = out.z = out.w = 0.0f;
    } else {  // Analyze: :152-172
        const Metrics m = metrics_from(q, N, st);
        out = make_float4(m.throughput, m.ttft, m.avg_token_time, m.rho);
    }
    g.req_out[slot] = out;
}

// Per-round reset of the device counters (one tiny kernel instead of two memsets; part of the captured round).
__global__ void sz2_round_reset(Sz2Args g) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        *g.n_req = 0;
        *g.n_live = 0;
    }
    if (i < 2 * kClasses + 1) g.ws.item_count[i] = 0;
}

// ---------------------------------------------------------------------------
// CreateAllocation (allocation.go:77-163) straight through, for one candidate.  Eval evaluates the points:
//   round(which, lo, hi, first)  the points of one round of the search `which` over (lo, hi): the two end points
//                                (first round only) and the midpoint tree of depth depth()
//   end(i), node(v)              {y, bail} of end point i / tree node v of the last round
//   solve(lambda, st)            Model.Solve for Analyze; false when it bailed
// Returns false when a consulted solve bailed (out is then nil).
//
// kStar: rateStar mode (the load grid) stops where the tail that reads the load starts (allocation.go:134), with
// out = nil or star_cand(rateStar).  Everything before that point (N from the tokens and srv_max_batch, the
// bisections, lambda*, rateStar = Analyze(lambda*).Throughput) does not read the load.
//
// kSearch: search mode (the SLO grid) runs only the search `which` at `target` and stops where it ends, with
// out = search_cand(SEARCH_NIL or SEARCH_OK, lambdaStar).  A search reads no other target: its bounds come from
// RateRange and its function is EvalTTFT or EvalITL (queueanalyzer.go:204-228, utils.go:26-70).
// ---------------------------------------------------------------------------
template <bool kStar, bool kSearch = false, class Eval>
__device__ __forceinline__ bool create_allocation(const DevFleet& f, int s, int a, int N, int K, float s1, float sN,
                                                  Eval& ev, Cand& out, int which = 0, float target = 0.0f) {
    out = cand_nil();
    if constexpr (kSearch) {
        SzStart b = sz_start(f, s, K, s1, sN);
        if (K < 2 || b.lmin > b.lmax) return true;
        SzSearch S{b.lmin, b.lmax, 0.0f, 0, 0, false};
        ev.round(which, S.lo, S.hi, true);
        int r = sz_ends(S, target, [&](int i) { return ev.end(i); });
        while (r == SZ_MORE) {
            r = sz_walk(S, target, ev.depth(), [&](int v) { return ev.node(v); });
            if (r == SZ_MORE) ev.round(which, S.lo, S.hi, false);
        }
        if (r == SZ_BAIL) return false;
        if (S.ind >= 0) out = search_cand(SEARCH_OK, S.xs);
        return true;
    }
    const SzStart b = sz_start(f, s, K, s1, sN);
    if (b.nil) return true;
    float xs_ttft = b.lmax, xs_itl = b.lmax;  // lambdaStar when a target is disabled (queueanalyzer.go:205,218)
    for (int w = 0; w < 2; ++w) {
        const float target = w == 0 ? f.srv_slo_ttft[s] : f.srv_slo_itl[s];
        if (!(target > 0.0f)) continue;
        SzSearch S{b.lmin, b.lmax, 0.0f, 0, 0, false};
        ev.round(w, S.lo, S.hi, true);
        int r = sz_ends(S, target, [&](int i) { return ev.end(i); });
        while (r == SZ_MORE) {
            r = sz_walk(S, target, ev.depth(), [&](int v) { return ev.node(v); });
            if (r == SZ_MORE) ev.round(w, S.lo, S.hi, false);
        }
        if (r == SZ_BAIL) return false;
        if (S.ind < 0) return true;
        (w == 0 ? xs_ttft : xs_itl) = S.xs;
    }
    float lam;
    ModelStats st;
    if (!sz_lambda(f, s, b.rmax, xs_ttft, xs_itl, lam)) return true;
    if (!ev.solve(lam, st)) return false;
    const float rate_star = metrics_from(ev.q, N, st).throughput;
    if constexpr (kStar) {
        out = star_cand(rate_star);
        return true;
    }
    SzReplicas r;
    if (!sz_replicas(f, s, a, b.rmax, rate_star, total_rate_of(f, s), r, lam)) return true;
    if (!ev.solve(lam, st)) return false;
    const Metrics m = metrics_from(ev.q, N, st);
    out = sz_cand(a, N, r, rate_star, m.ttft, m.avg_token_time, m.rho);
    return true;
}

// ---------------------------------------------------------------------------
// Small fleets (BASELINE configs[0]: one VariantAutoscaling = one candidate): ONE warp per candidate runs
// create_allocation in one launch — the same speculative midpoint trees as the rounds, but evaluated by the warp's
// lanes (round one: the two end points + 15 midpoints = 4 iterations; later rounds: 31 midpoints = 5 iterations)
// and read with warp shuffles.  No rounds, no sort, no host round trip: a reconcile of a handful of variants is
// three launches (trivial, this, unlimited argmin) instead of sixty.  Every lane computes the same decisions.
// ---------------------------------------------------------------------------
struct WarpEval {
    const double* tab;
    QParams q;
    int N, K, lane;
    bool first;
    float y;  // this lane's point
    int bail;
    __device__ __forceinline__ int depth() const { return first ? 4 : 5; }
    __device__ __forceinline__ void round(int which, float lo, float hi, bool first_round) {
        first = first_round;
        // this lane's point: round one = {lo, hi, nodes 1..15}, later rounds = nodes 1..31
        const bool has = first ? lane < 17 : lane < 31;
        float x = first && lane == 1 ? hi : lo;
        if (has && !(first && lane < 2)) x = sz_node_value(first ? lane - 1 : lane + 1, lo, hi);
        y = 0.0f;
        bail = 0;
        ModelStats st;
        if (has && !solve(x, st)) bail = 1;
        else if (has) y = target_value(q, which, N, st);
        __syncwarp();
    }
    __device__ __forceinline__ SzPt at(int src) const {
        return SzPt{__shfl_sync(0xffffffffu, y, src), __shfl_sync(0xffffffffu, bail, src) != 0};
    }
    __device__ __forceinline__ SzPt end(int i) const { return at(i); }
    __device__ __forceinline__ SzPt node(int v) const { return at(first ? v + 1 : v - 1); }
    __device__ __forceinline__ bool solve(float lambda, ModelStats& st) const {
        return SharedSolve{}(tab, N, K, lambda, st);
    }
};

template <bool kStar, bool kSearch = false>
__device__ __forceinline__ void size_warp(const SizeArgs& g, const SearchCols& sc = SearchCols{}) {
    const int j = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (j >= g.n_cand) return;
    const DevFleet& f = g.f;
    const int pair = g.cand_pair[j], s = pair / f.A, a = pair % f.A;
    const int N = g.cand_N[j], K = N + N * f.ratio;
    WarpEval ev;
    ev.tab = g.tab + 4 * g.tab_off[j];
    ev.q = qparams_of(f, s, a);
    ev.N = N;
    ev.K = K;
    ev.lane = lane;
    Cand c;
    bool ok;
    if constexpr (kSearch)
        ok = create_allocation<kStar, true>(f, s, a, N, K, (float)ev.tab[0], (float)ev.tab[4 * (N - 1)], ev, c,
                                            sc.which[j], sc.target[j]);
    else
        ok = create_allocation<kStar>(f, s, a, N, K, (float)ev.tab[0], (float)ev.tab[4 * (N - 1)], ev, c);
    if (lane == 0) {
        if (!ok) fb_push(g.fb, (unsigned)j);
        store_cand(g.cand, g.place.record(j, pair), c);
    }
}
__global__ void __launch_bounds__(128) size_warp_kernel(SizeArgs g) { size_warp<false>(g); }
__global__ void __launch_bounds__(128) size_warp_star(SizeArgs g) { size_warp<true>(g); }
__global__ void __launch_bounds__(128) size_warp_search(SearchArgs a) { size_warp<false, true>(a.g, a.search); }

// ---------------------------------------------------------------------------
// Stored-vector re-run of the candidates that bailed: one thread per candidate evaluates exactly the reference's
// points, one at a time, with the literal restatement solve_stored on its scratch slot.
// ---------------------------------------------------------------------------
struct StoredEval {
    StoredSolve stored;
    const double* tab;
    QParams q;
    int N, K;
    int which;
    float lo, hi;
    __device__ __forceinline__ int depth() const { return 1; }
    __device__ __forceinline__ void round(int w, float l, float h, bool) {
        which = w;
        lo = l;
        hi = h;
    }
    __device__ __forceinline__ SzPt at(float x) {
        ModelStats st;
        if (!solve(x, st)) return SzPt{0.0f, true};
        return SzPt{target_value(q, which, N, st), false};
    }
    __device__ __forceinline__ SzPt end(int i) { return at(i ? hi : lo); }
    __device__ __forceinline__ SzPt node(int) { return at(sz_mid(lo, hi)); }
    __device__ __forceinline__ bool solve(float lambda, ModelStats& st) { return stored(tab, N, K, lambda, st); }
};

// A candidate whose re-run fails is stored nil, as the drivers store a candidate that bailed, and returns the
// solve's code; in search mode it is stored SEARCH_FAIL instead and the call's status is left to the SLO grid's tail.
template <bool kStar, bool kSearch = false>
__device__ __forceinline__ void size_fallback_body(const SizeArgs& g, const FbRun& r,
                                                   const SearchCols& sc = SearchCols{}) {
    const DevFleet& f = g.f;
    fb_rerun(r, [&](unsigned long long item, double* p) {
        const int j = (int)item;
        const int pair = g.cand_pair[j], s = pair / f.A, a = pair % f.A;
        const int N = g.cand_N[j];
        StoredEval ev;
        ev.stored.p = p;
        ev.tab = g.tab + 4 * g.tab_off[j];
        ev.q = qparams_of(f, s, a);
        ev.N = N;
        ev.K = N + N * f.ratio;
        Cand c;
        bool ok;
        if constexpr (kSearch)
            ok = create_allocation<kStar, true>(f, s, a, N, ev.K, (float)ev.tab[0], (float)ev.tab[4 * (N - 1)], ev, c,
                                                sc.which[j], sc.target[j]);
        else
            ok = create_allocation<kStar>(f, s, a, N, ev.K, (float)ev.tab[0], (float)ev.tab[4 * (N - 1)], ev, c);
        int rc = ok ? 0 : ev.stored.rc;
        if (kSearch && !ok) {
            c = search_cand(SEARCH_FAIL, 0.0f);
            rc = 0;
        }
        store_cand(g.cand, g.place.record(j, pair), c);
        return rc;
    });
}
__global__ void size_fallback(SizeArgs g, FbRun r) { size_fallback_body<false>(g, r); }
__global__ void size_fallback_star(SizeArgs g, FbRun r) { size_fallback_body<true>(g, r); }
__global__ void size_fallback_search(SearchArgs sa, FbRun r) { size_fallback_body<false, true>(sa.g, r, sa.search); }

// ---------------------------------------------------------------------------
// The load grid's tail (allocation.go:134-163) at every level of a caller-given load list: one lane per (candidate,
// level) item whose level rate is a load (not negative, not zero; NaN and +Inf included).  The candidates are the
// load pairs in descending N with their rateStar from the rateStar mode above, which does not read the load.  Items
// are candidate-major (item e * L + l), so a warp reads the tables of one or a few pairs; a work counter hands out
// warps, as in sweep_kernel.  The final per-replica rate totalRate / replicas is at most rateStar, so a pair's
// chains are bounded by its lambda* chain.  Record (l * S + s) * A + a of the candidate block.
// ---------------------------------------------------------------------------
struct LoadArgs {
    DevFleet f;
    const int* cand_pair;       // [n_cand] pair ids sorted by descending N
    const int* cand_N;          // [n_cand]
    const long long* tab_off;   // [n_cand] entry offset of the candidate's table (N entries)
    const double* tab;
    const uint8_t* star_ok;     // [S * A] by pair: rateStar mode's records (0: nil at every load level) ...
    const float* rate_star;     // ... and their rateStar
    const float* level_rpm;     // [L * S] arrival rate of server s at level l (req/min)
    int n_cand, L;
    unsigned* counter;
    AllocCols cand;             // [L * S * A]
    FbList fb;                  // items that bailed: fb_pack(candidate, level)
};

// Candidate e's record at totalRate total_rate(s) (nil, or the feasible allocation); solve(tab, N, K, lambda, st)
// is Model.Solve for the final Analyze.  Returns false when that solve bailed (out is then nil).
template <class Total, class Solve>
__device__ __forceinline__ bool load_tail(const LoadArgs& g, int e, Total&& total_rate, Solve&& solve, Cand& out) {
    const DevFleet& f = g.f;
    const int pair = g.cand_pair[e], s = pair / f.A, a = pair % f.A, N = g.cand_N[e];
    const double* tab = g.tab + 4 * g.tab_off[e];
    out = cand_nil();
    if (!g.star_ok[pair]) return true;
    const float rate_star = g.rate_star[pair];
    SzReplicas r;
    float lam;
    if (!sz_replicas(f, s, a, rate_max_of((float)tab[4 * (N - 1)]), rate_star, total_rate(s), r, lam)) return true;
    ModelStats st;
    if (!solve(tab, N, N + N * f.ratio, lam, st)) return false;
    const Metrics m = metrics_from(qparams_of(f, s, a), N, st);
    out = sz_cand(a, N, r, rate_star, m.ttft, m.avg_token_time, m.rho);
    return true;
}

// The record of item fb_pack(e, l) in the level blocks: (l * S + s) * A + a, where s * A + a is candidate e's pair.
__device__ __forceinline__ size_t level_record(const DevFleet& f, const int* cand_pair, unsigned long long item) {
    const int e = (int)(item >> 32), l = (int)(unsigned)item;
    return (size_t)l * f.S * f.A + cand_pair[e];
}
// totalRate of server s at level l, for load_tail
struct LevelRate {
    const LoadArgs& g;
    int l;
    __device__ __forceinline__ float operator()(int s) const { return total_rate_of(at_level(g.f, g.level_rpm, l), s); }
};

// The tails' work loop: each warp takes the next 32 items from the work counter until all n_items are handed out,
// and lane i of a warp runs fn(item) on its item (lanes past n_items idle).
template <class Fn>
__device__ __forceinline__ void for_each_warp_item(unsigned* counter, unsigned n_items, Fn&& fn) {
    const int lane = threadIdx.x & 31;
    for (;;) {
        unsigned w = 0;
        if (lane == 0) w = atomicAdd(counter, 1u);
        w = __shfl_sync(0xffffffffu, w, 0);
        if ((unsigned long long)w * 32 >= n_items) break;
        const unsigned i = w * 32 + lane;
        if (i < n_items) fn(i);
    }
}

// The two sides of every tail.  A tail evaluates a packed item, eval(item, solve, out): false when a solve bailed
// (out is then nil); eval.record(item) is the index of its record.  The streaming side runs it with SharedSolve,
// appends the item to fb on a bail and stores the record either way; the re-run runs it with StoredSolve and stores
// the record only when every solve succeeded, else returns the failed solve's code.
template <class Eval>
__device__ __forceinline__ void tail_item(const FbList& fb, const AllocCols& cand, unsigned long long item,
                                          const Eval& eval) {
    Cand c;
    if (!eval(item, SharedSolve{}, c)) fb_push(fb, item);
    store_cand(cand, eval.record(item), c);
}
template <class Eval>
__device__ __forceinline__ void tail_rerun(const FbRun& r, const AllocCols& cand, const Eval& eval) {
    fb_rerun(r, [&](unsigned long long item, double* p) {
        StoredSolve solve{p, 0};
        Cand c;
        if (!eval(item, solve, c)) return solve.rc;
        store_cand(cand, eval.record(item), c);
        return 0;
    });
}

// The load grid's item fb_pack(e, l): candidate e at level l.
struct LoadTail {
    const LoadArgs& g;
    template <class Solve>
    __device__ __forceinline__ bool operator()(unsigned long long item, Solve&& solve, Cand& out) const {
        return load_tail(g, (int)(item >> 32), LevelRate{g, (int)(unsigned)item}, solve, out);
    }
    __device__ __forceinline__ size_t record(unsigned long long item) const {
        return level_record(g.f, g.cand_pair, item);
    }
};

__global__ void __launch_bounds__(256) load_kernel(LoadArgs g) {
    const DevFleet& f = g.f;
    const unsigned n_items = (unsigned)g.n_cand * (unsigned)g.L;  // <= S * A * L < 2^31
    for_each_warp_item(g.counter, n_items, [&](unsigned i) {
        const int e = (int)(i / (unsigned)g.L), l = (int)(i - (unsigned)e * g.L);
        const float rpm = g.level_rpm[(size_t)l * f.S + g.cand_pair[e] / f.A];
        // a level without load keeps trivial_kernel's nil / zero-load record
        if (!(rpm < 0.0f) && rpm != 0.0f) tail_item(g.fb, g.cand, fb_pack(e, l), LoadTail{g});
    });
}

// Stored-vector re-run of the items load_kernel bailed on.
__global__ void load_fallback(LoadArgs g, FbRun r) { tail_rerun(r, g.cand, LoadTail{g}); }

// ---------------------------------------------------------------------------
// The SLO grid's tail (DESIGN.md §3.11): CreateAllocation of every load pair at every level of a caller-given list
// of (ITL, TTFT, TPS) target rows, from the search records of search mode above.  A search reads only its own
// target, so phase 1 ran each distinct (server, search, target) once per load pair; this kernel combines a level's
// two records and runs the rest: lambda* (min with the TPS rule), rateStar = Analyze(lambda*).Throughput, the
// replicas at the level's totalRate and the final Analyze.  One lane per (candidate, level) item, candidate-major
// (item e * L + l), warps from a work counter, as in load_kernel.  Record (l * S + s) * A + a.
//
// The reference runs the ITL search only after the TTFT search succeeded, and phase 1 runs every key regardless.
// So a SEARCH_FAIL record fails the call only where the level's reference would have consulted it: a TTFT search
// always, an ITL search when the TTFT search is disabled or succeeded.
// ---------------------------------------------------------------------------
struct SloArgs {
    DevFleet f;
    const int* cand_pair;       // [n_cand] load pairs sorted by descending N
    const int* cand_N;          // [n_cand]
    const long long* tab_off;   // [n_cand] entry offset of the candidate's table (N entries)
    const double* tab;
    const float* slo_itl;       // [L * S] the targets of server s at level l
    const float* slo_ttft;
    const float* slo_tps;
    const int* key;             // [2 * L * S] the search key of (level, server, search) (l * S + s) * 2 + which
    AllocCols srch;             // [n_keys * A] search records by key * A + a (search_cand)
    int n_cand, L;
    unsigned* counter;
    int* status;                // set where a consulted search did not terminate
    AllocCols cand;             // [L * S * A]
    FbList fb;                  // items that bailed: fb_pack(candidate, level)
};

// The fleet as the SLO grid sees it at level l: the targets are row l of the level lists.
__device__ __forceinline__ DevFleet at_slo_level(const SloArgs& g, int l) {
    DevFleet fl = g.f;
    fl.srv_slo_itl = g.slo_itl + (size_t)l * g.f.S;
    fl.srv_slo_ttft = g.slo_ttft + (size_t)l * g.f.S;
    fl.srv_slo_tps = g.slo_tps + (size_t)l * g.f.S;
    return fl;
}

// CreateAllocation of pair (s, a) of f (the fleet at one level or tick: its targets, rate and tokens) from phase 1's
// search records: the sign gate, the level's two search records (key[kb + w] * A + a, where w = 0: TTFT, 1: ITL),
// lambda* (min with the TPS rule), rateStar = Analyze(lambda*).Throughput, the replicas at f's totalRate and the
// final Analyze.  tab is the pair's N-entry table; solve is Model.Solve for the two Analyze calls.  Returns false
// when a solve bailed (out is then nil).  The SLO grid and the SLO trace share it.
template <class Solve>
__device__ __forceinline__ bool slo_tail(const DevFleet& f, int s, int a, int N, const double* tab, const int* key,
                                         size_t kb, const AllocCols& srch, int* status, Solve&& solve, Cand& out) {
    const int K = N + N * f.ratio;
    out = cand_nil();
    const SzStart b = sz_start(f, s, K, (float)tab[0], (float)tab[4 * (N - 1)]);
    if (b.nil) return true;
    float xs[2] = {b.lmax, b.lmax};  // lambdaStar when a target is disabled (queueanalyzer.go:205,218)
    for (int w = 0; w < 2; ++w) {
        const float target = w == 0 ? f.srv_slo_ttft[s] : f.srv_slo_itl[s];
        if (!(target > 0.0f)) continue;
        const size_t k = (size_t)key[kb + w] * f.A + a;
        const int st = srch.feasible[k];
        if (st == SEARCH_FAIL) {
            atomicExch(status, 1);
            return true;
        }
        if (st == SEARCH_NIL) return true;
        xs[w] = srch.max_rate[k];
    }
    float lam;
    ModelStats st;
    if (!sz_lambda(f, s, b.rmax, xs[0], xs[1], lam)) return true;
    if (!solve(tab, N, K, lam, st)) return false;
    const QParams q = qparams_of(f, s, a);
    const float rate_star = metrics_from(q, N, st).throughput;
    SzReplicas r;
    if (!sz_replicas(f, s, a, b.rmax, rate_star, total_rate_of(f, s), r, lam)) return true;
    if (!solve(tab, N, K, lam, st)) return false;
    const Metrics m = metrics_from(q, N, st);
    out = sz_cand(a, N, r, rate_star, m.ttft, m.avg_token_time, m.rho);
    return true;
}

// The SLO grid's item fb_pack(e, l): candidate e at level l.
struct SloTail {
    const SloArgs& g;
    __device__ __forceinline__ size_t record(unsigned long long item) const {
        return level_record(g.f, g.cand_pair, item);
    }
    template <class Solve>
    __device__ __forceinline__ bool operator()(unsigned long long item, Solve&& solve, Cand& out) const {
        const int e = (int)(item >> 32), l = (int)(unsigned)item;
        const DevFleet f = at_slo_level(g, l);
        const int pair = g.cand_pair[e], s = pair / f.A;
        return slo_tail(f, s, pair % f.A, g.cand_N[e], g.tab + 4 * g.tab_off[e], g.key, ((size_t)l * f.S + s) * 2,
                        g.srch, g.status, solve, out);
    }
};

__global__ void __launch_bounds__(256) slo_kernel(SloArgs g) {
    const unsigned n_items = (unsigned)g.n_cand * (unsigned)g.L;  // <= S * A * L < 2^31
    for_each_warp_item(g.counter, n_items, [&](unsigned i) {
        const int e = (int)(i / (unsigned)g.L), l = (int)(i - (unsigned)e * g.L);
        tail_item(g.fb, g.cand, fb_pack(e, l), SloTail{g});
    });
}

// Stored-vector re-run of the items slo_kernel bailed on.
__global__ void slo_fallback(SloArgs g, FbRun r) { tail_rerun(r, g.cand, SloTail{g}); }

// ---------------------------------------------------------------------------
// The workload grid's tail (DESIGN.md §3.12): the load grid's tail (load_tail) on the key fleet, whose row k is
// server key_srv[k] at one (in_tokens, out_tokens) pair; phase 1 sized its load pairs k * A + a in rateStar mode.
// One lane per (key candidate, level that uses the key) item: candidate e's items are item_off[e] ..
// item_off[e + 1] - 1, and its j-th item is the j-th level of its key (lev[lev_off[k] + j]).  So items are
// candidate-major and a warp reads the tables of one or a few candidates; a work counter hands out warps, as in
// load_kernel.  totalRate is the level's rate over 60, or with a TPS target TPS over the key's out_tokens, which
// are the level's.  Record (l * S + s) * A + a.
// ---------------------------------------------------------------------------
struct WorkloadArgs {
    LoadArgs ld;           // phase 1 on the key fleet; level_rpm [L * S] by server and cand [L * S * A]
    const int* key_srv;    // [K] the key's server
    const int* lev_off;    // [K + 1] key k's levels are lev[lev_off[k] .. lev_off[k + 1]), ascending
    const int* lev;
    const int* item_off;   // [n_cand + 1] candidate e's first item
    int S;                 // servers of the fleet (ld.f.S counts the keys)
    int n_items;           // item_off[n_cand]: at most one per loaded (level, server, accelerator), < 2^31
};

// Item i's candidate e (the last one with item_off[e] <= i) and level l.
__device__ __forceinline__ void workload_item(const WorkloadArgs& g, int i, int& e, int& l) {
    int lo = 0, hi = g.ld.n_cand - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (g.item_off[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    e = lo;
    const int k = g.ld.cand_pair[e] / g.ld.f.A;
    l = g.lev[g.lev_off[k] + (i - g.item_off[e])];
}

// The workload grid's item fb_pack(e, l): candidate e at level l, from workload_item.
struct WorkloadTail {
    const WorkloadArgs& g;
    template <class Solve>
    __device__ __forceinline__ bool operator()(unsigned long long item, Solve&& solve, Cand& out) const {
        const int e = (int)(item >> 32), l = (int)(unsigned)item;
        const int k = g.ld.cand_pair[e] / g.ld.f.A;
        const float rpm = g.ld.level_rpm[(size_t)l * g.S + g.key_srv[k]];
        return load_tail(g.ld, e, [&](int) { return total_rate_of(g.ld.f, k, rpm); }, solve, out);
    }
    // record (l * S + s) * A + a of the key's server s
    __device__ __forceinline__ size_t record(unsigned long long item) const {
        const int pair = g.ld.cand_pair[item >> 32], l = (int)(unsigned)item;
        return ((size_t)l * g.S + g.key_srv[pair / g.ld.f.A]) * g.ld.f.A + pair % g.ld.f.A;
    }
};

__global__ void __launch_bounds__(256) workload_kernel(WorkloadArgs g) {
    for_each_warp_item(g.ld.counter, (unsigned)g.n_items, [&](unsigned i) {
        int e, l;
        workload_item(g, (int)i, e, l);
        tail_item(g.ld.fb, g.ld.cand, fb_pack(e, l), WorkloadTail{g});
    });
}

// Stored-vector re-run of the items workload_kernel bailed on.
__global__ void workload_fallback(WorkloadArgs g, FbRun r) { tail_rerun(r, g.ld.cand, WorkloadTail{g}); }

// ---------------------------------------------------------------------------
// The SLO trace's tail (DESIGN.md §3.17): the SLO grid's tail (slo_tail) on the workload trace's key fleet, whose row
// k is server key_srv[k] at one (in_tokens, out_tokens) pair.  Phase 1 ran each distinct (key row, search, target
// bits) once per load pair of the row, in search mode.  One lane per (key candidate, tick of its key row) item,
// located as workload_item locates them, warps from a work counter.  Item (e, t) evaluates the pair at f_t, the
// resident fleet with the rate, tokens and targets of row t (the key row's tokens are row t's), with the search
// records of tick t.  Record (t * S + s) * A + a.
// ---------------------------------------------------------------------------
struct SloTraceArgs {
    WorkloadArgs w;            // the key rows, their ticks and candidates, and the tables (w.ld, on the key fleet)
    DevFleet f;                // the resident fleet
    const int* tick_in;        // [L * S] row t of in_tokens and out_tokens (w.ld.level_rpm: of arrival_rpm)
    const int* tick_out;
    const float* slo_itl;      // [L * S] row t of the targets
    const float* slo_ttft;
    const float* slo_tps;
    const int* key;            // [2 * L * S] the search key of (tick, server, search) (t * S + s) * 2 + which
    AllocCols srch;            // search records by key * A + a (search_cand)
    int* status;               // set where a consulted search did not terminate
};

// f_t: the resident fleet with row t of the six row lists.
__device__ __forceinline__ DevFleet at_tick(const SloTraceArgs& g, int t) {
    const size_t o = (size_t)t * g.f.S;
    DevFleet ft = g.f;
    ft.srv_arrival_rpm = g.w.ld.level_rpm + o;
    ft.srv_in_tokens = g.tick_in + o;
    ft.srv_out_tokens = g.tick_out + o;
    ft.srv_slo_itl = g.slo_itl + o;
    ft.srv_slo_ttft = g.slo_ttft + o;
    ft.srv_slo_tps = g.slo_tps + o;
    return ft;
}

// The SLO trace's item fb_pack(e, t): key candidate e at tick t, from workload_item.
struct SloTraceTail {
    const SloTraceArgs& g;
    __device__ __forceinline__ size_t record(unsigned long long item) const { return WorkloadTail{g.w}.record(item); }
    template <class Solve>
    __device__ __forceinline__ bool operator()(unsigned long long item, Solve&& solve, Cand& out) const {
        const int e = (int)(item >> 32), t = (int)(unsigned)item;
        const int pair = g.w.ld.cand_pair[e], s = g.w.key_srv[pair / g.f.A];
        return slo_tail(at_tick(g, t), s, pair % g.f.A, g.w.ld.cand_N[e], g.w.ld.tab + 4 * g.w.ld.tab_off[e], g.key,
                        ((size_t)t * g.f.S + s) * 2, g.srch, g.status, solve, out);
    }
};

__global__ void __launch_bounds__(256) slo_trace_kernel(SloTraceArgs g) {
    for_each_warp_item(g.w.ld.counter, (unsigned)g.w.n_items, [&](unsigned i) {
        int e, t;
        workload_item(g.w, (int)i, e, t);
        tail_item(g.w.ld.fb, g.w.ld.cand, fb_pack(e, t), SloTraceTail{g});
    });
}

// Stored-vector re-run of the items slo_trace_kernel bailed on.
__global__ void slo_trace_fallback(SloTraceArgs g, FbRun r) { tail_rerun(r, g.w.ld.cand, SloTraceTail{g}); }

// ---------------------------------------------------------------------------
// SLO bounds (DESIGN.md §3.18): per (load pair, search), the two breakpoints in the target at which BinarySearch's
// boundary checks change their verdict.  Those checks read the target and y0 = eval(lambda_min), y1 =
// eval(lambda_max), and EvalTTFT and EvalITL come from one Model.Solve, so two solves per pair give both searches'
// bounds for every target.  bounds_tail solves one item fb_pack(candidate, end) per (pair, end), end 1 (lambda_max,
// the pair's longest chain) for every candidate first, and bounds_kernel classifies each (pair, search).
// ---------------------------------------------------------------------------
struct BoundsOut {  // [S * A * 2] by (s * A + a) * 2 + which
    uint8_t* kind;
    float *y_lo, *y_hi, *b1, *b2;
};
enum { BOUNDS_UNREAD = 0, BOUNDS_NIL = 1, BOUNDS_RISING = 2, BOUNDS_FALLING = 3 };

struct BoundsArgs {
    DevFleet f;
    const int* cand_pair;       // [n_cand] load pairs sorted by descending N
    const int* cand_N;          // [n_cand]
    const long long* tab_off;   // [n_cand] entry offset of the candidate's table (N entries)
    const double* tab;
    const int* cand_of_pair;    // [S * A] the pair's candidate, -1: not a load pair
    int n_cand;
    unsigned* counter;
    AllocCols ends;             // [2 * n_cand] record 2e + end: feasible 1 once solved (ttft / itl: the two
                                // metrics), 2 where no solve runs, 0 where the solve did not terminate
    FbList fb;                  // items that bailed: fb_pack(candidate, end)
    BoundsOut out;
};

// Candidate e's bisection bounds and whether its boundary solves run: not for K < 2 (sz_start's nil), an empty
// range (BinarySearch's error before any evaluation) or lambda_min < 0, where Model.Solve marks the model invalid
// (queuemodel.go:27-37) and the first evaluation fails.  Every other model of K >= 2 states is valid: rho = 1 - p[0]
// of the previous solve lies in [0, 1] (NaN passes the check).
__device__ __forceinline__ bool bounds_range(const BoundsArgs& g, int e, float& lmin, float& lmax, bool& nil) {
    const int N = g.cand_N[e], K = N + N * g.f.ratio;
    const double* tab = g.tab + 4 * g.tab_off[e];
    float rmax;
    sz_range((float)tab[0], (float)tab[4 * (N - 1)], rmax, lmin, lmax);
    nil = lmin > lmax || lmin < 0.0f;
    return K >= 2;
}

// Item fb_pack(e, end): Model.Solve(lambda, 1) at lambda = lambda_min (end 0) or lambda_max (end 1), in req/ms as
// BinarySearch evaluates them, then EvalTTFT and EvalITL (target_value) from that one solve.
struct BoundsTail {
    const BoundsArgs& g;
    __device__ __forceinline__ size_t record(unsigned long long item) const {
        return 2 * (size_t)(item >> 32) + (unsigned)item;
    }
    template <class Solve>
    __device__ __forceinline__ bool operator()(unsigned long long item, Solve&& solve, Cand& out) const {
        const int e = (int)(item >> 32), end = (int)(unsigned)item;
        out = cand_nil();
        float lmin, lmax;
        bool nil;
        if (!bounds_range(g, e, lmin, lmax, nil) || nil) {
            out.feasible = 2;
            return true;
        }
        const int pair = g.cand_pair[e], N = g.cand_N[e], K = N + N * g.f.ratio;
        ModelStats st;
        if (!solve(g.tab + 4 * g.tab_off[e], N, K, end ? lmax : lmin, st)) return false;
        const QParams q = qparams_of(g.f, pair / g.f.A, pair % g.f.A);
        out.feasible = 1;
        out.ttft = target_value(q, 0, N, st);
        out.itl = target_value(q, 1, N, st);
        return true;
    }
};

__global__ void __launch_bounds__(256) bounds_tail(BoundsArgs g) {
    const unsigned n = (unsigned)g.n_cand;  // 2 * n < 2^31 (n <= S * A)
    for_each_warp_item(g.counter, 2 * n, [&](unsigned i) {
        tail_item(g.fb, g.ends, i < n ? fb_pack((int)i, 1) : fb_pack((int)(i - n), 0), BoundsTail{g});
    });
}

// Stored-vector re-run of the items bounds_tail bailed on.
__global__ void bounds_fallback(BoundsArgs g, FbRun r) { tail_rerun(r, g.ends, BoundsTail{g}); }

// The class of target t for a search with boundary values y0, y1, decided by sz_ends itself over the stand-in range
// (lo, hi) = (0, 1): NIL where it ends with ind -1, FREE where it ends at hi, SEARCHED where it ends at lo with ind
// 0 or bisects.  As a rank that never decreases as t grows (DESIGN.md §3.18): rising (y0 < y1) NIL 0, SEARCHED 1,
// FREE 2; otherwise FREE 0, SEARCHED 1, NIL 2.
__device__ __forceinline__ int bounds_rank(float y0, float y1, bool rising, float t) {
    SzSearch S{0.0f, 1.0f, 0.0f, 0, 0, false};
    const int r = sz_ends(S, t, [&](int i) { return SzPt{i ? y1 : y0, false}; });
    const int cls = r == SZ_MORE ? 1 : (S.ind < 0 ? 0 : (S.xs == S.hi ? 2 : 1));  // NIL 0, SEARCHED 1, FREE 2
    return rising ? cls : 2 - cls;
}
// The smallest positive float32 target (bits 1 .. 0x7f800000 = +Inf) of rank >= k, or NaN when +Inf's rank is
// below k: a bisection over the bit patterns.
__device__ __forceinline__ float bounds_first(float y0, float y1, bool rising, int k) {
    const unsigned inf = 0x7f800000u;
    const auto reaches = [&](unsigned bits) { return bounds_rank(y0, y1, rising, __uint_as_float(bits)) >= k; };
    if (!reaches(inf)) return __uint_as_float(0x7fc00000u);
    if (reaches(1u)) return __uint_as_float(1u);
    return __uint_as_float(bits_first(1u, inf, reaches));
}

// One thread per (pair, search) entry (s * A + a) * 2 + which.
__global__ void __launch_bounds__(256) bounds_kernel(BoundsArgs g) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2ll * g.f.S * g.f.A) return;
    const int which = (int)(i & 1), e = g.cand_of_pair[i >> 1];
    int kind = BOUNDS_UNREAD;
    float y0 = 0.0f, y1 = 0.0f, b1 = 0.0f, b2 = 0.0f;
    float lmin, lmax;
    bool nil;
    if (e >= 0 && bounds_range(g, e, lmin, lmax, nil)) {
        kind = BOUNDS_NIL;
        if (!nil) {
            const AllocCols& r = g.ends;
            y0 = which ? r.itl[2 * (size_t)e] : r.ttft[2 * (size_t)e];
            y1 = which ? r.itl[2 * (size_t)e + 1] : r.ttft[2 * (size_t)e + 1];
            const bool rising = y0 < y1;
            kind = rising ? BOUNDS_RISING : BOUNDS_FALLING;
            b1 = bounds_first(y0, y1, rising, 1);
            b2 = bounds_first(y0, y1, rising, 2);
        }
    }
    if (g.out.kind) g.out.kind[i] = (uint8_t)kind;
    if (g.out.y_lo) g.out.y_lo[i] = y0;
    if (g.out.y_hi) g.out.y_hi[i] = y1;
    if (g.out.b1) g.out.b1[i] = b1;
    if (g.out.b2) g.out.b2[i] = b2;
}

// ---------------------------------------------------------------------------
// Load intervals (DESIGN.md §3.10): per server, the float32 arrival rates in [lo, hi] at which the load grid's
// winner changes its decision key (feasible, acc, replicas, batch, cost, value, max_rate).  Above zero load a load
// pair's key is a function of its state (nrep, gate), and that state never decreases as the rate grows, so each
// pair's next change is the first float32 at which a monotone predicate flips: a bisection over the bit patterns.
// interval_kernel walks the union of the pairs' steps with one warp per server and emits an interval wherever the
// winner's key changes; interval_tail then runs the load grid's tail (load_tail) at every interval start whose
// winner is a load pair, and interval_fallback re-runs the items it bailed on.
// ---------------------------------------------------------------------------
// What the walks (the load intervals and the load margins) and their tails share.
struct WalkArgs {
    LoadArgs ld;               // phase 1's candidates and rateStar records (level_rpm, L and cand unused)
    const int* cand_of_pair;   // [S * A] the pair's index in ld's candidate list, -1: not a load candidate
    const float* lo;           // the windows (req/min), one row of S per level
    const float* hi;
    AllocCols rec;             // the records
    FbList items;              // the tail's work list: fb_pack(accelerator, record)
    int* status;               // set when a window holds a rate at which a pair has 0 replicas (see iv_advance)
};

struct IntervalArgs : WalkArgs {  // one row of windows; rec [S * M]
    int M;                     // intervals per server
    int* count;                // [S]
    uint8_t* truncated;        // [S]
    float* start;              // [S * M]
};

// A pair's state at one rate: the key is a function of (nrep, gate), and over marks a replica count beyond
// INT32_MAX (the int32 column and go_f64_to_int's wrap end the monotone part there).  gate: 0 the final rate is
// not positive, 1 Analyze accepts it, 2 it is above RateRange.Max.
struct IvState {
    long long nrep;
    int gate;
    bool over;
    __device__ bool operator!=(const IvState& o) const { return nrep != o.nrep || gate != o.gate || over != o.over; }
};

// What one accelerator of the warp's server decides at the current point, and where that changes next.
struct IvAcc {
    Cand key;       // the load grid's record at the point without its latency columns; value = TransitionPenalty
    float next;     // the smallest rate above the point at which the state changes (+Inf: none up to hi)
    float rate_star, rmax;
    int N;
    int tail;       // 1: a load pair, whose record needs the tail (the latency columns) at an interval start
    bool over;
};
// The host sizes interval_kernel's and margin_kernel's warps per block from this (64 A and 68 A bytes per warp), and
// the tests place their accelerator counts on those layout thresholds.
static_assert(sizeof(IvAcc) == 64, "IvAcc layout");

__device__ __forceinline__ IvState iv_state(const DevFleet& f, int s, int a, const IvAcc& p, float rpm, Cand* key) {
    const float total = total_rate_of(f, s, rpm);
    SzReplicas r;
    float lam;
    const bool ok = sz_replicas(f, s, a, p.rmax, p.rate_star, total, r, lam);
    IvState st;
    st.nrep = r.nrep;
    st.gate = ok ? 1 : (sz_final_rate(total, r.nrep) <= 0.0f ? 0 : 2);
    st.over = !(sz_quotient(total, p.rate_star) <= 2147483647.0);
    if (key) {
        *key = cand_nil();
        if (ok) {
            *key = sz_cand(a, p.N, r, p.rate_star, 0.0f, 0.0f, 0.0f);
            key->value = penalty_of(f, s, *key);
        }
    }
    return st;
}

// Narrows a bisection for pred's first hold in (l, h] to the +-64-ulp bracket around est's float32 when pred fails at
// the bracket's bottom (or that is l) and holds at its top (or that is h, where top_known says it holds).  Returns
// whether it did; a bracket that does not check out leaves (l, h] alone, so the bisection finds the same point.
template <class Pred>
__device__ __forceinline__ bool ulp_bracket(double est, bool top_known, unsigned& l, unsigned& h, Pred&& pred) {
    const unsigned e = __float_as_uint(__double2float_rn(est));
    const unsigned bl = e > l && e - l > 64 ? e - 64 : l, bh = e < h && h - e > 64 ? e + 64 : h;
    if (est < 3.0e38 && bl < bh && (bl == l || !pred(bl)) && ((top_known && bh == h) || pred(bh))) {
        l = bl;
        h = bh;
        return true;
    }
    return false;
}

// Accelerator a of server s at rate x (x = 0 or in (0, hi]): its key and its next step.  The window of x is row
// `row` of the bound lists g.lo / g.hi (the load intervals have one row).  f is the fleet the key is taken on: g.ld.f,
// or on a margin call the row's view (mg_view).  k is the row of g.ld that phase 1 sized the pair on: s, or on a
// workload margin call the row's token key.  With hi = x it returns right after the key.
__device__ __forceinline__ void iv_advance(const WalkArgs& g, const DevFleet& f, int row, int s, int k, int a,
                                           float x, float hi, IvAcc& p) {
    const float inf = __int_as_float(0x7f800000);
    // the class at x: pair_class reads only whether the rate is negative or zero, and lo is 0 when x = 0
    const int cls = pair_class(at_level(f, x == 0.0f ? g.lo : g.hi, row), s, a, true);
    p.tail = 0;
    p.over = false;
    p.next = x == 0.0f && hi > 0.0f ? __int_as_float(1) : inf;  // rpm = 0 is a point of its own
    if (cls != PAIR_LOAD) {
        p.key = cand_nil();
        if (cls == PAIR_ZERO) {
            p.key = zero_load_alloc(f, s, a);
            p.key.value = penalty_of(f, s, p.key);
        }
        return;
    }
    const int e = g.cand_of_pair[k * f.A + a];
    if (!g.ld.star_ok[k * f.A + a]) {  // nil at every load
        p.key = cand_nil();
        return;
    }
    p.tail = 1;
    p.N = g.ld.cand_N[e];
    p.rate_star = g.ld.rate_star[k * f.A + a];
    p.rmax = rate_max_of((float)g.ld.tab[4 * (g.ld.tab_off[e] + p.N - 1)]);
    const IvState at = iv_state(f, s, a, p, x, &p.key);
    p.over = at.over;
    // totalRate rounds to 0 below 60 * 2^-150 req/min: with min_replicas 0 the pair has 0 replicas and Analyze
    // solves at 0/0, whose rescale loop does not terminate, so the load grid fails at this rate; so does the call
    if (at.nrep == 0) *g.status = 1;
    if (f.srv_slo_tps[s] != 0.0f || at.over) return;  // a TPS target: totalRate does not read the load
    // the first float32 in (x, hi] whose state differs from x's: the state is non-decreasing in the rate (nrep
    // first, then gate at a fixed nrep, with over absorbing), so "differs" is a monotone predicate
    auto differs = [&](unsigned bits) { return iv_state(f, s, a, p, __uint_as_float(bits), nullptr) != at; };
    unsigned l = __float_as_uint(x), h = __float_as_uint(hi);
    if (h <= l) return;
    // The step is within a few ulps of 60 * nrep * rateStar (the count grows) or 60 * nrep * RateRange.Max (the
    // rate check starts rejecting): bisect in the bracket around the nearer estimate when it holds the step;
    // otherwise over the whole range, when that holds one.
    bool bracketed = false;
    if (at.nrep >= 1 && at.gate != 0) {
        double est = 60.0 * (double)at.nrep * (double)p.rate_star;
        if (at.gate == 1) est = fmin(est, 60.0 * (double)at.nrep * (double)p.rmax);
        bracketed = ulp_bracket(est, false, l, h, differs);
    }
    if (!bracketed && !differs(h)) return;
    p.next = __uint_as_float(bits_first(l, h, differs));
}

// SolveUnlimited over the warp's accelerators: strict '<' from MaxFloat32, ties to the lower accelerator id.
// Returns the winner's accelerator (-1: none) on every lane.
__device__ __forceinline__ int iv_winner(const IvAcc* acc, int A, int lane) {
    float v = 3.40282346638528859811704183484516925440e+38f;
    int w = -1;
    for (int a = lane; a < A; a += 32)
        if (acc[a].key.feasible && acc[a].key.value < v) {
            v = acc[a].key.value;
            w = a;
        }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, d);
        const int ow = __shfl_xor_sync(0xffffffffu, w, d);
        if (ow >= 0 && (w < 0 || ov < v || (ov == v && ow < w))) {
            v = ov;
            w = ow;
        }
    }
    return w;
}

// The decision key's columns, bitwise.
__device__ __forceinline__ bool iv_same_key(const Cand& x, const Cand& y) {
    return x.feasible == y.feasible && x.acc == y.acc && x.replicas == y.replicas && x.batch == y.batch &&
           __float_as_uint(x.cost) == __float_as_uint(y.cost) && __float_as_uint(x.value) == __float_as_uint(y.value) &&
           __float_as_uint(x.max_rate) == __float_as_uint(y.max_rate);
}

// The warp's least and greatest v.
__device__ __forceinline__ float warp_fmin(float v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, d));
    return v;
}
__device__ __forceinline__ float warp_fmax(float v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, d));
    return v;
}

// One step up the union of the warp's pair steps: nx, the least next step of the warp's accelerators, and where
// nx <= hi the pairs that step there advanced to it (advance(a, nx)), after which `over` is set on every lane when
// some pair of the warp is over.  Returns nx.
template <class Advance>
__device__ __forceinline__ float iv_step(const IvAcc* acc, int A, int lane, float hi, bool& over, Advance&& advance) {
    float nx = __int_as_float(0x7f800000);
    for (int a = lane; a < A; a += 32) nx = fminf(nx, acc[a].next);
    nx = warp_fmin(nx);
    if (!(nx <= hi)) return nx;
    __syncwarp();
    for (int a = lane; a < A; a += 32)
        if (acc[a].next == nx) {
            advance(a, nx);
            over |= acc[a].over;
        }
    __syncwarp();
    over = __any_sync(0xffffffffu, over);
    return nx;
}

// One warp per server; the accelerators' state lives in dynamic shared memory (A entries per warp).
__global__ void __launch_bounds__(128) interval_kernel(IntervalArgs g) {
    extern __shared__ IvAcc iv_acc[];
    const DevFleet& f = g.ld.f;
    const int A = f.A, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int s = blockIdx.x * (blockDim.x >> 5) + wid;
    if (s >= f.S) return;
    IvAcc* acc = iv_acc + (size_t)wid * A;
    const float hi = g.hi[s];
    float x = g.lo[s];
    auto advance = [&](int a, float y) { iv_advance(g, f, 0, s, s, a, y, hi, acc[a]); };
    bool truncated = false;
    for (int a = lane; a < A; a += 32) {
        advance(a, x);
        truncated |= acc[a].over;
    }
    __syncwarp();
    int n = 0;
    truncated = __any_sync(0xffffffffu, truncated);  // a pair needs more than INT32_MAX replicas at lo
    Cand prev = cand_nil();
    while (!truncated) {
        const int w = iv_winner(acc, A, lane);
        const Cand key = w >= 0 ? acc[w].key : cand_nil();
        if (n == 0 || !iv_same_key(key, prev)) {
            if (n == g.M) {
                truncated = true;
                break;
            }
            if (lane == 0) {
                const size_t r = (size_t)s * g.M + n;
                g.start[r] = x;
                if (w >= 0 && acc[w].tail) fb_push(g.items, fb_pack(w, (int)r));
                else store_cand(g.rec, r, key);
            }
            prev = key;
            ++n;
        }
        // the list ends below the first rate that overflows
        const float nx = iv_step(acc, A, lane, hi, truncated, advance);
        if (!(nx <= hi)) break;
        x = nx;
    }
    if (lane == 0) {
        g.count[s] = n;
        g.truncated[s] = truncated;
    }
}

// Item fb_pack(a, r) of a walk's work list: record r, whose winner is the load pair of accelerator a of server s,
// sized on row k of g.ld (see iv_advance), is the load grid's tail at rate x, then the value against the fleet
// fleet() returns.
// Priced: phase 1 sized the pair at another price or AccCount (the profile margins' key fleet), so the record is
// first priced at fleet()'s (priced_at).
template <bool Priced = false, class Fleet, class Solve>
__device__ __forceinline__ bool walk_load_tail(const WalkArgs& g, unsigned long long item, int s, int k, float x,
                                               Fleet&& fleet, Solve&& solve, Cand& out) {
    const DevFleet& f = g.ld.f;
    const int a = (int)(item >> 32), e = g.cand_of_pair[k * f.A + a];
    if (!load_tail(g.ld, e, [&](int) { return total_rate_of(f, k, x); }, solve, out)) return false;
    if constexpr (Priced) {
        const DevFleet& fl = fleet();
        out = priced_at(fl, fl.srv_model[s], a, out);
        if (out.feasible) out.value = penalty_of(fl, s, out);
    } else {
        if (out.feasible) out.value = penalty_of(fleet(), s, out);
    }
    return true;
}

// A walk's tail kernel: eval over the work list, grid-stride.
template <class Eval>
__device__ __forceinline__ void walk_tail(const WalkArgs& g, const Eval& eval) {
    const int n = min(*g.items.count, g.items.cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        tail_item(g.ld.fb, g.rec, g.items.item[i], eval);
}

// The record r at an interval start.
struct IvTail {
    const IntervalArgs& g;
    template <class Solve>
    __device__ __forceinline__ bool operator()(unsigned long long item, Solve&& solve, Cand& out) const {
        const int r = (int)(unsigned)item, s = r / g.M;
        return walk_load_tail(g, item, s, s, g.start[r], [&]() -> const DevFleet& { return g.ld.f; }, solve, out);
    }
    __device__ __forceinline__ size_t record(unsigned long long item) const { return (unsigned)item; }
};

__global__ void __launch_bounds__(256) interval_tail(IntervalArgs g) { walk_tail(g, IvTail{g}); }

// Stored-vector re-run of the interval starts interval_tail bailed on.
__global__ void interval_fallback(IntervalArgs g, FbRun r) { tail_rerun(r, g.rec, IvTail{g}); }

// ---------------------------------------------------------------------------
// Load margins (DESIGN.md §3.19): per (level, server), the stretch of float32 rates in the window [lo, hi] around
// the level's rate r on which the load grid's winner keeps its decision key.  margin_kernel runs one warp per
// (level, server) and walks up from r as interval_kernel walks (iv_advance) to the first change of the winner's key.
// Then it walks down: a pair's state at x holds on a stretch [start, x], found by one bisection, because the state
// never decreases as the rate grows.  The warp maximum y of the starts is the next rate below which some pair
// changes, and the walk stops at the first such y whose float below changes the key.  margin_tail then runs the load
// grid's tail at the records (at r, below lo, at hi) whose winner is a load pair, and margin_fallback re-runs the
// items it bailed on.
//
// On a trace (DESIGN.md §3.21, the kernels' Trace instantiations) level t is tick t, solved against the current
// allocation c_t that the workload trace carries into it.  margin_chain writes c_t of every (tick, server) first, and
// every read of the current allocation then goes through the row's view of the fleet (mg_view).
//
// The workload margins (DESIGN.md §3.22) give each row its own tokens.  The kernels then take a TokenMarginArgs:
// phase 1 sized the rows' token keys, so ld.f is the key fleet and item i's pairs are those of its key row key[i];
// the resident fleet is f, and every read of a server's rate, tokens or current allocation goes through the row's
// view, which carries the row's tokens.  The kernels exist once per Trace, overloaded on the argument type, so the
// load-only calls' kernels keep their names and code.
//
// The profile margins (DESIGN.md §3.23) also give each row its own acc_cost and perf_* columns: a ProfileMarginArgs,
// whose row view adds them (profile_at), whose keys are per (item, accelerator) with a perf column (mg_pair), and
// whose tail records, sized on the key fleet, are priced at the row before their value.
//
// The SLO margins (DESIGN.md §3.24) give each row its own ITL, TTFT and TPS targets: an SloMarginArgs, whose row view
// adds them, so that pair_class, iv_state's totalRate and mg_start's TPS test read row l's.  Its keys are the
// workload margins' refined by the targets' bits, one per item, and the key fleet carries each key's targets.
// ---------------------------------------------------------------------------
enum { MG_LO_OPEN = 1, MG_HI_OPEN = 2, MG_TRUNCATED = 4 };  // the header's WVA_MARGIN_*

struct MarginArgs : WalkArgs {  // windows [n]; rec [3 * n]: at (k = 0), below (1), above (2), record k * n + i
    const float* rate;         // [n] the levels' rates, index l * S + s (req/min)
    int n;                     // L * S, with 3 * n < 2^31
    float* lo_out;             // [n]
    float* hi_out;             // [n]
    uint8_t* flags;            // [n]
    int* cur_acc;              // [n] on a trace: c_t of item t * S + s, written by margin_chain (unused otherwise)
    int* cur_replicas;
    float* cur_cost;
};

struct TokenMarginArgs : MarginArgs {  // ld: phase 1 on the key fleet, one row per (server, in, out) key
    DevFleet f;                // the resident fleet
    const int* key;            // [n] item i's key row in ld, -1: none (window top 0, or tokens that are no load)
    const int* in_tokens;      // [n] the rows' tokens, index l * S + s
    const int* out_tokens;
};

struct ProfileMarginArgs : TokenMarginArgs {  // ld: phase 1 on the profile calls' key fleet
    DevFleet rows;             // acc_cost and perf_* at row 0: the caller's row lists, or f's own columns ...
    unsigned per_level;        // ... bit c (0: acc_cost, 1 .. 8: perf_* in list order) set: column c is a row list
    const int* pair_key;       // [n * A] item i's key row in ld for accelerator a, -1: none; NULL: key[i] for every a
};

struct SloMarginArgs : TokenMarginArgs {  // ld: phase 1 on the key fleet, one row per (server, tokens, targets) key
    const float* slo_itl;      // [n] the rows' targets, index l * S + s
    const float* slo_ttft;
    const float* slo_tps;
};

// A key that names one row of ld for every accelerator of the item (the load and workload margins), or item i's row
// per accelerator (the profile margins: pair_key, or key[i] for every accelerator without a perf column).  The
// profile key holds the item, not a pointer, so that margin_kernel keeps to its registers.
struct MgPairKey {
    const ProfileMarginArgs& g;
    int i;
};
__device__ __forceinline__ int mg_pair(int k, int) { return k; }
__device__ __forceinline__ int mg_pair(const MgPairKey& k, int a) {
    return k.g.pair_key ? k.g.pair_key[(size_t)k.i * k.g.f.A + a] : k.g.key[k.i];
}

// The resident fleet; item i's key in ld (phase 1's records), for server s; and row l's fleet without c_t.
__device__ __forceinline__ const DevFleet& mg_fleet(const MarginArgs& g) { return g.ld.f; }
__device__ __forceinline__ const DevFleet& mg_fleet(const TokenMarginArgs& g) { return g.f; }
__device__ __forceinline__ int mg_key(const MarginArgs&, int, int s) { return s; }
__device__ __forceinline__ int mg_key(const TokenMarginArgs& g, int i, int) { return g.key[i]; }
__device__ __forceinline__ MgPairKey mg_key(const ProfileMarginArgs& g, int i, int) { return MgPairKey{g, i}; }
__device__ __forceinline__ const DevFleet& mg_row(const MarginArgs& g, int) { return g.ld.f; }
__device__ __forceinline__ DevFleet mg_row(const TokenMarginArgs& g, int l) {
    return at_rows(g.f, LoadRows{nullptr, g.in_tokens, g.out_tokens}, l);
}
// ... and with row l's acc_cost and perf_* columns (profile_at)
__device__ __forceinline__ DevFleet mg_row(const ProfileMarginArgs& g, int l) {
    return at_rows(profile_at(g, l), LoadRows{nullptr, g.in_tokens, g.out_tokens}, l);
}
// ... and with row l's ITL, TTFT and TPS targets
__device__ __forceinline__ DevFleet mg_row(const SloMarginArgs& g, int l) {
    DevFleet fl = at_rows(g.f, LoadRows{nullptr, g.in_tokens, g.out_tokens}, l);
    const size_t o = (size_t)l * g.f.S;
    fl.srv_slo_itl = g.slo_itl + o;
    fl.srv_slo_ttft = g.slo_ttft + o;
    fl.srv_slo_tps = g.slo_tps + o;
    return fl;
}

// The fleet of row l: on a trace with the current allocation c_t of tick t = l.
template <bool Trace, class Args>
__device__ __forceinline__ DevFleet mg_view(const Args& g, int l) {
    DevFleet ft = mg_row(g, l);
    if constexpr (Trace) {
        const size_t o = (size_t)l * mg_fleet(g).S;
        ft.srv_cur_acc = g.cur_acc + o;
        ft.srv_cur_replicas = g.cur_replicas + o;
        ft.srv_cur_cost = g.cur_cost + o;
    }
    return ft;
}

// The trace's chain: one warp per server walks the ticks with c_t in registers (c_0 from the fleet), lanes over the
// accelerators as in margin_kernel.  At tick t it stores c_t, takes every pair's key at the tick's rate against c_t
// (iv_advance with hi = the rate, which returns after the key) and the winner (iv_winner: strict '<' from MaxFloat32,
// ties to the lower accelerator id); c_{t+1} is the winner's (acc, replicas, cost) when there is one, c_t otherwise
// (Server.ApplyDesiredAlloc).  Those key columns are the ones margin_tail writes into `at`, so the chain needs no
// latency solve.  Launched with up to 128 threads; A IvAcc states per warp in dynamic shared memory.
template <class Args>
__device__ __forceinline__ void mg_chain(const Args& g) {
    extern __shared__ IvAcc iv_acc[];
    const DevFleet& f = mg_fleet(g);
    const int A = f.A, S = f.S, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int s = blockIdx.x * (blockDim.x >> 5) + wid;
    if (s >= S) return;
    IvAcc* acc = iv_acc + (size_t)wid * A;
    int cur_acc = f.srv_cur_acc[s], cur_replicas = f.srv_cur_replicas[s];
    float cur_cost = f.srv_cur_cost[s];
    const int L = g.n / S;
    for (int t = 0; t < L; ++t) {
        const int i = t * S + s;
        if (lane == 0) {
            g.cur_acc[i] = cur_acc;
            g.cur_replicas[i] = cur_replicas;
            g.cur_cost[i] = cur_cost;
        }
        __syncwarp();  // c_t is visible to the warp, and the previous tick's reads of acc are done
        const DevFleet ft = mg_view<true>(g, t);
        const auto k = mg_key(g, i, s);
        const float r = g.rate[i];
        for (int a = lane; a < A; a += 32) iv_advance(g, ft, t, s, mg_pair(k, a), a, r, r, acc[a]);
        __syncwarp();
        const int w = iv_winner(acc, A, lane);
        if (w >= 0) {
            cur_acc = acc[w].key.acc;
            cur_replicas = acc[w].key.replicas;
            cur_cost = acc[w].key.cost;
        }
    }
}
__global__ void __launch_bounds__(128) margin_chain(MarginArgs g) { mg_chain(g); }
__global__ void __launch_bounds__(128) margin_chain(TokenMarginArgs g) { mg_chain(g); }
__global__ void __launch_bounds__(128) margin_chain(ProfileMarginArgs g) { mg_chain(g); }
__global__ void __launch_bounds__(128) margin_chain(SloMarginArgs g) { mg_chain(g); }

// nextafterf(x, 0) for x > 0
__device__ __forceinline__ float mg_below(float x) { return __uint_as_float(__float_as_uint(x) - 1u); }

// Accelerator a of server s at rate x in (0, r], where bottom is the window's smallest positive rate: its key at x
// and the smallest rate in [bottom, x] at which its state is its state at x.  A pair that is not a load pair, or
// one with a TPS target, has one key at every positive rate (iv_advance set it at r).
__device__ __forceinline__ float mg_start(const DevFleet& f, int s, int a, IvAcc& p, float x, float bottom) {
    if (!p.tail) return bottom;
    const IvState at = iv_state(f, s, a, p, x, &p.key);
    if (f.srv_slo_tps[s] != 0.0f) return bottom;
    // "same state as at x" is false below the start and true from it on up to x: a monotone predicate
    auto same = [&](unsigned bits) { return !(iv_state(f, s, a, p, __uint_as_float(bits), nullptr) != at); };
    unsigned l = __float_as_uint(bottom), h = __float_as_uint(x);
    if (h <= l || same(l)) return bottom;
    // !same(l), same(h).  The start is within a few ulps of 60 * (nrep - 1) * rateStar (the count reached nrep) or,
    // at a rate the check rejects, 60 * nrep * RateRange.Max (the rejection started): bisect in the bracket around
    // that estimate when it holds the start, otherwise over the whole range.
    if (at.nrep >= 1 && at.gate != 0) {
        double est = 60.0 * (double)(at.nrep - 1) * (double)p.rate_star;
        if (at.gate == 2) est = fmax(est, 60.0 * (double)at.nrep * (double)p.rmax);
        ulp_bracket(est, true, l, h, same);
    }
    return __uint_as_float(bits_first(l, h, same));
}

// Accelerator a of server s at rate 0 of row `row` (the window's bottom lo = 0): its zero-load record or nil, as
// iv_advance sets it there.
__device__ __forceinline__ void mg_at_zero(const DevFleet& f, const float* lo, int row, int s, int a, IvAcc& p) {
    const int cls = pair_class(at_level(f, lo, row), s, a, true);
    p.tail = 0;
    p.key = cand_nil();
    if (cls == PAIR_ZERO) {
        p.key = zero_load_alloc(f, s, a);
        p.key.value = penalty_of(f, s, p.key);
    }
}

// Record k (0: at, 1: below, 2: above) of item i is winner w's record at the walk's point: a load pair's goes to
// margin_tail, any other is stored as it is (a zero-load record or nil).  Lane 0 calls it.
__device__ __forceinline__ void mg_emit(const MarginArgs& g, int k, int i, int w, const IvAcc* acc) {
    const int r = k * g.n + i;
    if (w >= 0 && acc[w].tail) fb_push(g.items, fb_pack(w, r));
    else store_cand(g.rec, r, w >= 0 ? acc[w].key : cand_nil());
}

// One warp per (level, server) item i = l * S + s; the accelerators' IvAcc states, then their stretch starts, live
// in dynamic shared memory (A entries of each per warp).  Launched with up to 128 threads; with
// __launch_bounds__(128) ptxas keeps it at 72 registers and spills, with room for 96 it uses 80 and does not.
// Trace: level l is tick l, on the fleet mg_view(g, l).
template <bool Trace, class Args>
__device__ __forceinline__ void mg_walk(const Args& g) {
    constexpr bool Rows = Trace || !std::is_same<Args, MarginArgs>::value;  // f is a row view, not g.ld.f
    extern __shared__ IvAcc iv_acc[];
    const int A = mg_fleet(g).A, lane = threadIdx.x & 31, wid = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const int i = blockIdx.x * wpb + wid;
    if (i >= g.n) return;
    const int l = i / mg_fleet(g).S, s = i - l * mg_fleet(g).S;
    const auto k = mg_key(g, i, s);
    DevFleet ft;
    if constexpr (Rows) ft = mg_view<Trace>(g, l);
    const DevFleet& f = Rows ? ft : g.ld.f;
    IvAcc* acc = iv_acc + (size_t)wid * A;
    float* start = (float*)(iv_acc + (size_t)wpb * A) + (size_t)wid * A;
    const float r = g.rate[i], lo = g.lo[i], hi = g.hi[i];
    const float inf = __int_as_float(0x7f800000);
    auto advance = [&](int a, float x) { iv_advance(g, f, l, s, mg_pair(k, a), a, x, hi, acc[a]); };
    bool over = false;
    for (int a = lane; a < A; a += 32) {
        advance(a, r);
        over |= acc[a].over;
    }
    __syncwarp();
    // The load intervals over the window visit its smallest positive rate, where a min_replicas-0 pair may have 0
    // replicas; the call refuses the window as they do (r = 0 steps there first, see below).
    const float bottom = lo > 0.0f ? lo : __int_as_float(1);
    if (r > 0.0f && bottom < r)
        for (int a = lane; a < A; a += 32)
            if (acc[a].tail && iv_state(f, s, a, acc[a], bottom, nullptr).nrep == 0) *g.status = 1;
    const int w0 = iv_winner(acc, A, lane);
    const Cand key = w0 >= 0 ? acc[w0].key : cand_nil();
    if (lane == 0) mg_emit(g, 0, i, w0, acc);
    int flags = 0;
    float lo_out = r, hi_out = r;
    if (__any_sync(0xffffffffu, over)) {
        flags = MG_TRUNCATED;  // a pair needs more than INT32_MAX replicas at r
    } else {
        // up: the union of the pairs' steps above r, as interval_kernel walks it
        for (;;) {
            const float nx = iv_step(acc, A, lane, hi, over, advance);
            if (!(nx <= hi)) {
                flags |= MG_HI_OPEN;
                hi_out = inf;
                break;
            }
            hi_out = nx;
            if (over) {  // the stretch ends below the first rate that overflows
                flags |= MG_TRUNCATED;
                break;
            }
            const int w = iv_winner(acc, A, lane);
            if (!iv_same_key(w >= 0 ? acc[w].key : cand_nil(), key)) {
                if (lane == 0) mg_emit(g, 2, i, w, acc);
                break;
            }
        }
        // down: from r to the first rate below which the key differs
        if (!(r > 0.0f)) {
            flags |= MG_LO_OPEN;  // r = 0 is the window's bottom
            lo_out = lo;
        } else {
            // Every pair's key and stretch at r first (x = y = r); then at each step down the pairs whose stretch
            // starts at y take their key and stretch at x, the float below y.  Below the smallest positive rate
            // lies rate 0, a point of its own.
            for (int a = lane; a < A; a += 32) start[a] = r;
            float x = r, y = r;
            for (;;) {
                const bool at_zero = !(x > 0.0f);
                __syncwarp();
                for (int a = lane; a < A; a += 32) {
                    if (at_zero) mg_at_zero(f, g.lo, l, s, a, acc[a]);
                    else if (start[a] == y) start[a] = mg_start(f, s, a, acc[a], x, bottom);
                }
                __syncwarp();
                if (x != r) {
                    const int w = iv_winner(acc, A, lane);
                    if (!iv_same_key(w >= 0 ? acc[w].key : cand_nil(), key)) {
                        lo_out = y;
                        if (lane == 0) mg_emit(g, 1, i, w, acc);
                        break;
                    }
                }
                y = bottom;
                for (int a = lane; a < A; a += 32) y = fmaxf(y, start[a]);
                y = warp_fmax(y);
                // no pair changes its state in [bottom, x]: the stretch reaches the window's bottom
                if (at_zero || (y == bottom && lo > 0.0f)) {
                    flags |= MG_LO_OPEN;
                    lo_out = lo;
                    break;
                }
                x = mg_below(y);
            }
        }
    }
    if (lane == 0) {
        g.lo_out[i] = lo_out;
        g.hi_out[i] = hi_out;
        g.flags[i] = (uint8_t)flags;
    }
}
template <bool Trace>
__global__ void __maxnreg__(96) margin_kernel(MarginArgs g) { mg_walk<Trace>(g); }
template <bool Trace>
__global__ void __maxnreg__(96) margin_kernel(TokenMarginArgs g) { mg_walk<Trace>(g); }
// The profile margins' row view holds eight more row pointers (acc_cost and the perf_* columns of row l) through the
// walk: at 96 registers ptxas spills 116 bytes, with room for 120 it uses 118 and does not (4 blocks of 128 threads
// per SM instead of 5).
template <bool Trace>
__global__ void __maxnreg__(120) margin_kernel(ProfileMarginArgs g) { mg_walk<Trace>(g); }
// The SLO margins' row view holds three more row pointers (the targets of row l) through the walk: at 96 registers
// ptxas spills 4 bytes in the grid's instantiation, with room for 104 it uses 100 and does not (4 blocks of 128
// threads per SM instead of 5); the trace's uses 96 either way.
template <bool Trace>
__global__ void __maxnreg__(104) margin_kernel(SloMarginArgs g) { mg_walk<Trace>(g); }

// The record r = k * n + i: record k of item i, at the record's rate (r, the float below lo_out, or hi_out), its
// value on a trace against c_t.  The profile margins' records are priced at their row and valued on its view.
template <bool Trace, class Args>
struct MgTail {
    const Args& g;
    template <class Solve>
    __device__ __forceinline__ bool operator()(unsigned long long item, Solve&& solve, Cand& out) const {
        const int r = (int)(unsigned)item, k = r / g.n, i = r - k * g.n, S = mg_fleet(g).S;
        const float x = k == 0 ? g.rate[i] : (k == 1 ? mg_below(g.lo_out[i]) : g.hi_out[i]);
        const int s = i % S, key = mg_pair(mg_key(g, i, s), (int)(item >> 32));
        if constexpr (std::is_same<Args, ProfileMarginArgs>::value)
            return walk_load_tail<true>(g, item, s, key, x, [&] { return mg_view<Trace>(g, i / S); }, solve, out);
        else if constexpr (Trace) return walk_load_tail(g, item, s, key, x, [&] { return mg_view<true>(g, i / S); }, solve, out);
        else return walk_load_tail(g, item, s, key, x, [&]() -> const DevFleet& { return mg_fleet(g); }, solve, out);
    }
    __device__ __forceinline__ size_t record(unsigned long long item) const { return (unsigned)item; }
};

template <bool Trace>
__global__ void __launch_bounds__(256) margin_tail(MarginArgs g) { walk_tail(g, MgTail<Trace, MarginArgs>{g}); }
template <bool Trace>
__global__ void __launch_bounds__(256) margin_tail(TokenMarginArgs g) {
    walk_tail(g, MgTail<Trace, TokenMarginArgs>{g});
}
template <bool Trace>
__global__ void __launch_bounds__(256) margin_tail(ProfileMarginArgs g) {
    walk_tail(g, MgTail<Trace, ProfileMarginArgs>{g});
}
template <bool Trace>
__global__ void __launch_bounds__(256) margin_tail(SloMarginArgs g) { walk_tail(g, MgTail<Trace, SloMarginArgs>{g}); }

// Stored-vector re-run of the records margin_tail bailed on.
template <bool Trace>
__global__ void margin_fallback(MarginArgs g, FbRun r) { tail_rerun(r, g.rec, MgTail<Trace, MarginArgs>{g}); }
template <bool Trace>
__global__ void margin_fallback(TokenMarginArgs g, FbRun r) { tail_rerun(r, g.rec, MgTail<Trace, TokenMarginArgs>{g}); }
template <bool Trace>
__global__ void margin_fallback(ProfileMarginArgs g, FbRun r) {
    tail_rerun(r, g.rec, MgTail<Trace, ProfileMarginArgs>{g});
}
template <bool Trace>
__global__ void margin_fallback(SloMarginArgs g, FbRun r) { tail_rerun(r, g.rec, MgTail<Trace, SloMarginArgs>{g}); }

}  // namespace wva

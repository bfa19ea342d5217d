// wva_b200.cu — host engine + C ABI (include/wva_b200.h) over the sm_90a kernels.
//
// Host-side mirror of pkg/core.System / pkg/manager.Manager for the hot path: the fleet
// is packed once into a single device arena (one H2D copy), derived work lists
// (candidates ordered by queue size, shared service-rate tables) are cached on the
// handle, every call enqueues its kernels on the handle's stream and ends with one D2H
// copy of the result block.  There is no CPU compute fallback: without a CUDA device
// wva_create fails.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <numeric>
#include <optional>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/wva_b200.h"
#include "wva_kernels.cuh"
#include "wva_size.cuh"

using namespace wva;

namespace {

// Growable buffers that own their memory: freed when the handle that holds them is deleted.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
};
struct PinBuf {
    void* p = nullptr;
    size_t cap = 0;
    PinBuf() = default;
    PinBuf(const PinBuf&) = delete;
    PinBuf& operator=(const PinBuf&) = delete;
    ~PinBuf() {
        if (p) cudaFreeHost(p);
    }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
};

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Columns packed into one buffer, each starting on an `align`-byte boundary (an empty column still gets an
// address of its own).  The offsets take() and put() return hand out the device pointers.  take() records where a
// column with a host destination lies, so the layout and the copy-back cannot disagree.  put() lays out a column
// whose host bytes are src, and upload_tables copies every such column into the host image before its fill runs:
// src must stay alive, and must not be resized, until upload_tables returns.
struct Cols {
    struct Col {
        size_t off, bytes;
        void* dst;
    };
    struct Src {
        size_t off, bytes;
        const void* src;
    };
    size_t align, bytes = 0;
    std::vector<Col> out;  // the columns that have a host destination
    std::vector<Src> in;   // the columns copied verbatim from host memory
    explicit Cols(size_t a) : align(a) {}
    size_t take(size_t n, void* dst = nullptr) {
        const size_t at = bytes;
        if (dst) out.push_back({at, n, dst});
        bytes = align_up(at + std::max<size_t>(n, 1), align);
        return at;
    }
    size_t put(const void* src, size_t n) {
        const size_t at = take(n);
        if (n) in.push_back({at, n, src});
        return at;
    }
    // device buffer `dev` -> the destinations, enqueued on `st`
    cudaError_t copy_back(const void* dev, cudaStream_t st) const {
        for (const Col& c : out)
            if (c.bytes) {
                const cudaError_t e = cudaMemcpyAsync(c.dst, (const char*)dev + c.off, c.bytes, cudaMemcpyDeviceToHost, st);
                if (e != cudaSuccess) return e;
            }
        return cudaSuccess;
    }
    // host image of the buffer -> the destinations
    void scatter(const void* host) const {
        for (const Col& c : out)
            if (c.bytes) memcpy(c.dst, (const char*)host + c.off, c.bytes);
    }
};

// One allocation record on the host (the limited-mode solve works on these).
struct HostCand {
#define HOST_FIELD(name, type, required) type name;
    WVA_ALLOC_COLUMNS(HOST_FIELD)
#undef HOST_FIELD
};

// Host copy of the fleet columns (the caller's pointers are never retained).
struct HostFleet {
    int A = 0, T = 0, M = 0, S = 0;
#define HOST_COLUMN(abi, name, type, len) std::vector<type> name;
    WVA_FLEET_COLUMNS(HOST_COLUMN)
#undef HOST_COLUMN
    bool unlimited = true, delayed_best_effort = false;
    int saturation_policy = 0;
    wva_tunables tun{10, 0.1f};

    // gates of CreateAllocation + candidate rule (mirrors pair_class on the device)
    int pair_class(int s, int a, bool honour_keep) const { return pair_class(s, a, honour_keep, srv_arrival_rpm[s]); }
    // ... at the arrival rate rpm
    int pair_class(int s, int a, bool honour_keep, float rpm) const {
        const int m = srv_model[s];
        return pair_class(s, a, honour_keep, rpm, m >= 0 && m < M && perf_present[(size_t)m * A + a]);
    }
    // ... with `present` in place of the model's perf_present at a (the profile grid's rows)
    int pair_class(int s, int a, bool honour_keep, float rpm, bool present) const {
        return pair_class(s, a, honour_keep, rpm, srv_in_tokens[s], srv_out_tokens[s], srv_cur_acc[s], present);
    }
    // ... at a row's tokens in / out and current accelerator cur (a level's or a trace tick's)
    int pair_class(int s, int a, bool honour_keep, float rpm, int in, int out, int cur) const {
        const int m = srv_model[s];
        return pair_class(s, a, honour_keep, rpm, in, out, cur, m >= 0 && m < M && perf_present[(size_t)m * A + a]);
    }
    int pair_class(int s, int a, bool honour_keep, float rpm, int in, int out, int cur, bool present) const {
        if (honour_keep && srv_keep_acc[s] && cur != WVA_ACC_NONE && cur != a) return 0;
        if (rpm < 0.0f || in < 0 || out < 0) return 0;
        const int m = srv_model[s];
        if (m < 0 || m >= M) return 0;
        if (!present) return 0;
        if (!srv_has_target[s]) return 0;
        if (rpm == 0.0f || out == 0) return PAIR_ZERO;
        return PAIR_LOAD;
    }
    // batch size of a candidate: pkg/core/allocation.go:77-87, in Go's 64-bit int (the AtTokens rule can exceed int32)
    long long pair_batch(int s, int a) const {
        if (srv_max_batch[s] > 0) return srv_max_batch[s];
        const size_t k = (size_t)srv_model[s] * A + a;
        const long long t = (long long)perf_max_batch[k] * (long long)perf_at_tokens[k] / srv_out_tokens[s];
        return std::max<long long>(t, 1);
    }
    // The queue model of batch size N (at most 2^20) has N + N * ratio states.  The reference counts them in Go's
    // 64-bit int; the kernels, the fallback scratch and the int32 ABI count them in int32, so a model of 2^31
    // states or more is refused instead of being built at a wrapped size.
    bool queue_fits(long long N) const { return N * (1 + (long long)tun.max_queue_to_batch_ratio) < (1ll << 31); }
    // limited mode charges every allocation to its accelerator's type: each accelerator needs one
    bool every_acc_typed() const {
        for (int a = 0; a < A; ++a)
            if (T <= 0 || acc_type[a] < 0 || acc_type[a] >= T) return false;
        return true;
    }
};

struct Column {
    size_t off, bytes;
};

constexpr uint64_t kUncached = ~0ull;  // an epoch no fleet reaches

// One set of shared service-rate tables (build_pair_tables) and the device image of the lists that describe them:
// upload_tables() fills it, build_tables() builds the tables, and the caching rules are at upload_tables().
struct PairTables {
    DevBuf lists, tab, ls;  // the lists image; 4 doubles per entry; entries + n floats of prefix log2 sums
    // what the lists were uploaded for: epoch_tokens and the path's other inputs (kUncached: nothing to reuse)
    uint64_t epoch = kUncached;
    std::vector<int> key;
    int n = 0, len_max = 1;                   // tables, the longest one (1 when there are none)
    bool with_ls = false;                     // ls is built (the sweep needs none)
    size_t o_pair = 0, o_off = 0, o_len = 0;  // byte offsets in `lists` of the pair ids, entry offsets and lengths
    bool holds(uint64_t e, const std::vector<int>& k = {}) const { return epoch == e && key == k; }
    const int* pair() const { return (const int*)((const char*)lists.p + o_pair); }
    const long long* off() const { return (const long long*)((const char*)lists.p + o_off); }
    const int* len() const { return (const int*)((const char*)lists.p + o_len); }
};

}  // namespace

struct wva_handle {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_k0 = nullptr, ev_k1 = nullptr, ev_d0 = nullptr, ev_d1 = nullptr;
    std::string err;
    int64_t launches = 0;
    float last_kernel_ms = 0.f, last_device_ms = 0.f;

    // resident fleet
    bool resident = false;
    HostFleet hf;
    DevBuf arena;
    PinBuf stage;
    DevFleet df{};
    Column col_rate{}, col_in{}, col_out{};
    uint64_t epoch_tokens = 0;  // bumped when service-rate tables become stale

    // service-rate tables: one set per path, so that a size grid or a load grid never evicts wva_solve's; the
    // sweep builds into the grid's
    PairTables size_tabs, sg_tabs, lg_tabs, grid_tabs;

    // size path
    DevBuf d_sz_state, d_sz_req, d_sz_sort;
    PinBuf sz_pin;
    DevBuf d_lg_star;  // the load grid's rateStar records (shared with the load intervals)
    DevBuf d_iv;       // the load intervals' and load margins' output columns and work list
    DevBuf d_slo;      // the SLO grid's search records
    DevBuf d_prof;     // the profile grid's key records
    DevBuf d_price;    // the price thresholds
    DevBuf d_bounds;   // the SLO bounds' end records and entries

    // grid path
    DevBuf d_sort, d_best, d_pb, d_rows;
    // shared
    DevBuf d_cand_block, d_win_block, d_ctrl, d_fb_list[2], d_scratch, d_cells, d_sweep, d_dbg;
    // peer exchange of the winner block (multi-GPU, one process per GPU on one node)
    struct Xchg {
        int world = 0, rank = 0;
        size_t block_bytes = 0, slot_stride = 0;   // one gathered buffer = world * slot_stride bytes
        char* local = nullptr;                     // [2 parities][world slots] + flags, cudaMalloc'ed here
        size_t local_bytes = 0, flags_off = 0;
        std::vector<char*> peer;                   // base pointers of every rank's buffer (peer[rank] == local)
        char** d_peer = nullptr;
        unsigned long long epoch = 0;
        int* d_err = nullptr;
    } xchg;
    // the most recent solution (for wva_summarize): 0 none, 1 winner block on the device, 2 host copy (greedy)
    int last_kind = 0;
    std::vector<HostCand> last_win;
    DevBuf d_summary;
    bool dbg_cycles = false;
    const unsigned* dbg_plan = nullptr;
    size_t dbg_n = 0;
    PinBuf out_stage;

    int fail(int code, const char* what, cudaError_t e = cudaSuccess) {
        err = what;
        if (e != cudaSuccess) {
            err += ": ";
            err += cudaGetErrorString(e);
        }
        return code;
    }
};

#define CK(call)                                                              \
    do {                                                                      \
        cudaError_t _e = (call);                                              \
        if (_e != cudaSuccess) return h->fail(WVA_ERR_CUDA, #call, _e);       \
    } while (0)

namespace {


// control block on the device: a handful of ints
// CTRL_FB2_COUNT: a second fallback list of the same call (the load grid's tail items)
enum {
    CTRL_COUNTER = 0, CTRL_FB_COUNT = 1, CTRL_FB_STATUS = 2, CTRL_FB2_COUNT = 3, CTRL_FB_OVERFLOW = 4, CTRL_INTS = 8
};

// ---- SoA result blocks: the wva_allocs columns of n records, 16-byte aligned ----------------
struct Block {
    struct {
#define BLOCK_OFFSET(name, type, required) size_t name;
        WVA_ALLOC_COLUMNS(BLOCK_OFFSET)
#undef BLOCK_OFFSET
    } off;
    size_t bytes;
    size_t n;
};
Block block_layout(size_t n) {
    Block b;
    Cols c(16);
#define BLOCK_PLACE(name, type, required) b.off.name = c.take(sizeof(type) * n);
    WVA_ALLOC_COLUMNS(BLOCK_PLACE)
#undef BLOCK_PLACE
    b.bytes = c.bytes;
    b.n = n;
    return b;
}
AllocCols block_cols(void* base, const Block& b) {
    AllocCols c;
#define BLOCK_COL(name, type, required) c.name = (type*)((char*)base + b.off.name);
    WVA_ALLOC_COLUMNS(BLOCK_COL)
#undef BLOCK_COL
    return c;
}
void scatter_block(const void* host_block, const Block& b, const wva_allocs* out) {
    if (!out) return;
#define BLOCK_SCATTER(name, type, required) \
    if (out->name) memcpy(out->name, (const char*)host_block + b.off.name, sizeof(type) * b.n);
    WVA_ALLOC_COLUMNS(BLOCK_SCATTER)
#undef BLOCK_SCATTER
}
// Records [k * n, (k + 1) * n) of block b, as a block of n records (a call that returns several record lists in one
// block scatters each through its own view)
Block sub_block(const Block& b, size_t k, size_t n) {
    Block s = b;
#define SUB_OFFSET(name, type, required) s.off.name += sizeof(type) * k * n;
    WVA_ALLOC_COLUMNS(SUB_OFFSET)
#undef SUB_OFFSET
    s.n = n;
    return s;
}
AllocCols cols_from_abi(const wva_allocs* a) {
    AllocCols c{};
    if (!a) return c;
#define ABI_COL(name, type, required) c.name = a->name;
    WVA_ALLOC_COLUMNS(ABI_COL)
#undef ABI_COL
    return c;
}

// ---- fleet validation + upload ----------------------------------------------
// nullptr when the fleet is well formed, else what is wrong with it
const char* fleet_problem(const wva_fleet* f) {
    if (!f) return "fleet is NULL";
    if (f->n_acc < 0 || f->n_types < 0 || f->n_models < 0 || f->n_servers < 0) return "negative size in fleet";
    // a column of positive length must be there; the message names the column's group
    struct Len {
        long long n;
        const char* null_column;
    };
    const Len A{f->n_acc, "NULL accelerator column"}, T{f->n_types, "NULL capacity column"},
        MA{(long long)f->n_models * f->n_acc, "NULL perf column"}, S{f->n_servers, "NULL server column"};
#define NULL_CHECK(abi, name, type, len) \
    if (len.n > 0 && !f->abi) return len.null_column;
    WVA_FLEET_COLUMNS(NULL_CHECK)
#undef NULL_CHECK
    for (int a = 0; a < f->n_acc; ++a)
        if (f->n_types > 0 && (f->acc_type[a] < 0 || f->acc_type[a] >= f->n_types)) return "accelerator type id out of range";
    if (f->tun.max_queue_to_batch_ratio < 0) return "negative queue ratio";
    return nullptr;
}

// Host copy of every column (the caller's pointers are never retained).
void fill_host_fleet(HostFleet& hf, const wva_fleet* f) {
    const size_t A = f->n_acc, T = f->n_types, M = f->n_models, S = f->n_servers, MA = M * A;
    hf.A = (int)A; hf.T = (int)T; hf.M = (int)M; hf.S = (int)S;
#define FILL(abi, name, type, len) hf.name.assign(f->abi, f->abi + len);
    WVA_FLEET_COLUMNS(FILL)
#undef FILL
    hf.unlimited = f->unlimited != 0;
    hf.delayed_best_effort = f->delayed_best_effort != 0;
    hf.saturation_policy = f->saturation_policy;
    hf.tun = f->tun;
}

int upload_fleet(wva_handle* h, const wva_fleet* f) {
    if (const char* what = fleet_problem(f)) return h->fail(WVA_ERR_BAD_ARG, what);
    CK(cudaStreamSynchronize(h->stream));  // the pinned stage may still feed an earlier async copy
    HostFleet& hf = h->hf;
    fill_host_fleet(hf, f);

    // one arena in list order, one H2D copy
    Cols arena(256);
#define ARENA_PLACE(abi, name, type, len)                   \
    const size_t bytes_##name = sizeof(type) * hf.name.size(); \
    const Column c_##name{arena.take(bytes_##name), bytes_##name};
    WVA_FLEET_COLUMNS(ARENA_PLACE)
#undef ARENA_PLACE
    CK(h->arena.ensure(arena.bytes));
    CK(h->stage.ensure(arena.bytes));
    char* st = (char*)h->stage.p;
    const char* d = (const char*)h->arena.p;
    DevFleet& df = h->df;
#define ARENA_FILL(abi, name, type, len)                                         \
    if (c_##name.bytes) memcpy(st + c_##name.off, hf.name.data(), c_##name.bytes); \
    df.name = (const type*)(d + c_##name.off);
    WVA_FLEET_COLUMNS(ARENA_FILL)
#undef ARENA_FILL
    CK(cudaMemcpyAsync(h->arena.p, h->stage.p, arena.bytes, cudaMemcpyHostToDevice, h->stream));
    df.A = hf.A; df.T = hf.T; df.M = hf.M; df.S = hf.S;
    df.ratio = hf.tun.max_queue_to_batch_ratio;
    df.penalty = hf.tun.accel_penalty_factor;
    h->col_rate = c_srv_arrival_rpm; h->col_in = c_srv_in_tokens; h->col_out = c_srv_out_tokens;
    h->resident = true;
    h->epoch_tokens++;
    h->last_kind = 0;
    return WVA_OK;
}

int ensure_ctrl(wva_handle* h) {
    CK(h->d_ctrl.ensure(CTRL_INTS * sizeof(int)));
    CK(cudaMemsetAsync(h->d_ctrl.p, 0, CTRL_INTS * sizeof(int), h->stream));
    return WVA_OK;
}

// The stored-vector fallback (DESIGN.md §3.2): a call has up to two lists (the load grid's two phases), each with
// its own count and buffer, re-run by a fixed number of threads with one scratch slot each.
constexpr int kFbBlocks = 2, kFbThreads = 64, kFbSlots = kFbBlocks * kFbThreads;
constexpr int kFbCount[2] = {CTRL_FB_COUNT, CTRL_FB2_COUNT};

// List `list` (0 or 1) of up to cap entries, and the scratch for chains of batch size up to Nmax: the largest batch
// size of a model the call builds (0 when it builds none), which the caller has checked with queue_fits.  Called
// before the kernels that use them are enqueued: a DevBuf that grows frees its old memory, and cudaFree synchronises.
int prepare_fallback(wva_handle* h, int list, int cap, int Nmax, FbRun& r) {
    CK(h->d_fb_list[list].ensure(sizeof(unsigned long long) * std::max(cap, 1)));
    if (!h->hf.queue_fits(Nmax)) return h->fail(WVA_ERR_UNSUPPORTED, "queue model of 2^31 states or more");
    const int Kmax = (int)(Nmax * (1 + (long long)h->hf.tun.max_queue_to_batch_ratio));
    CK(h->d_scratch.ensure(sizeof(double) * ((size_t)Kmax + 1) * kFbSlots));
    int* ctrl = (int*)h->d_ctrl.p;
    r.list = FbList{ctrl + kFbCount[list], (unsigned long long*)h->d_fb_list[list].p, cap};
    r.scratch = (double*)h->d_scratch.p;
    r.Kmax = Kmax;
    r.status = ctrl + CTRL_FB_STATUS;
    r.overflow = ctrl + CTRL_FB_OVERFLOW;
    return WVA_OK;
}

// Enqueues kernel<<<grid, block, smem>>>(args...) with programmatic dependent launch: the kernel may start while the
// kernel before it in the stream runs, and reads nothing that kernel writes before its pdl_wait().
template <class... Params, class... Args>
int launch_pdl(wva_handle* h, void (*kernel)(Params...), unsigned grid, unsigned block, size_t smem, Args&&... args) {
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = h->stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    CK(cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
    h->launches++;
    return WVA_OK;
}

// Enqueues a re-run kernel (grid_fallback, size_fallback, ...) over r's list; with pdl, by launch_pdl (the kernel
// calls pdl_wait() first).
template <class Args>
int launch_fallback(wva_handle* h, void (*kernel)(Args, FbRun), const Args& g, const FbRun& r, bool pdl = false) {
    if (pdl) return launch_pdl(h, kernel, kFbBlocks, kFbThreads, 0, g, r);
    kernel<<<kFbBlocks, kFbThreads, 0, h->stream>>>(g, r);
    h->launches++;
    return WVA_OK;
}

// Enqueues kernel(args...) with one thread per record of an n_rec-record block (trivial_kernel, profile_kernel, ...).
// The overload of kernel is the one whose parameters are exactly the arguments' types.
template <class... Args>
void launch_records(wva_handle* h, long long n_rec, void (*kernel)(Args...), const Args&... args) {
    if (n_rec <= 0) return;
    kernel<<<(unsigned)((n_rec + 255) / 256), 256, 0, h->stream>>>(args...);
    h->launches++;
}

// Enqueues a tail kernel (load_kernel, slo_kernel, workload_kernel, sweep_kernel) whose warps take their items from
// a work counter: at most 8 blocks of 256 threads per SM, and no more than `warps` warps.  Then records ev_k1 (the
// call's kernel time ends with the tail) and re-runs the items it bailed on (fallback over fb).
template <class Args>
int launch_tail(wva_handle* h, void (*kernel)(Args), void (*fallback)(Args, FbRun), const Args& g, long long warps,
                const FbRun& fb) {
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, 0));
    per_sm = std::max(1, std::min(per_sm, 8));
    const unsigned blocks = (unsigned)std::min<long long>((long long)h->sm_count * per_sm, (warps + 7) / 8);
    kernel<<<blocks, 256, 0, h->stream>>>(g);
    h->launches++;
    CK(cudaEventRecord(h->ev_k1, h->stream));
    launch_fallback(h, fallback, g, fb);
    return WVA_OK;
}

// The (server, accelerator) pairs of hf that keep(s, a) accepts, as ids s * A + a with their batch sizes N, sorted
// by descending N (stable: equal N keep the pair order).
template <class Keep>
int sorted_pairs(wva_handle* h, const HostFleet& hf, Keep keep, std::vector<int>& pairs, std::vector<int>& N) {
    const int A = hf.A, S = hf.S;
    std::vector<int> Ns((size_t)S * A, 0);
    pairs.clear();
    for (int s = 0; s < S; ++s)
        for (int a = 0; a < A; ++a)
            if (keep(s, a)) {
                const long long n = hf.pair_batch(s, a);
                if (n > (1 << 20)) return h->fail(WVA_ERR_UNSUPPORTED, "batch size above 2^20");
                if (!hf.queue_fits(n))
                    return h->fail(WVA_ERR_UNSUPPORTED,
                                   "queue model of 2^31 states or more (batch size x (1 + max_queue_to_batch_ratio))");
                Ns[(size_t)s * A + a] = (int)n;
                pairs.push_back(s * A + a);
            }
    std::stable_sort(pairs.begin(), pairs.end(), [&](int x, int y) { return Ns[x] > Ns[y]; });
    N.resize(pairs.size());
    for (size_t j = 0; j < pairs.size(); ++j) N[j] = Ns[pairs[j]];
    return WVA_OK;
}

// ---- shared service-rate tables ---------------------------------------------
// Upload the lists of one set of tables: table t is pair[t]'s first len[t] service rates, in the caller's order,
// at entry offset len[0] + .. + len[t-1].  The columns the caller laid out in `c` come first in the same image:
// those put() there are copied in, then fill(host image) writes the rest; the table lists follow.  One H2D copy,
// then tab (and ls when with_ls) are sized.
// The instance is left keyed kUncached; a path that caches sets the key once its tables are built.
//
// Every entry point that takes a fleet calls upload_fleet, which bumps epoch_tokens, so only the resident calls can
// reuse lists.  Each path's rule:
// - solve path (size_tabs): lists and tables are rebuilt only when epoch_tokens changes.  A wva_update_load +
//   wva_resolve (or wva_resolve_device) tick with unchanged tokens and pair classes uploads nothing and launches
//   no build_pair_tables.
// - size grid (sg_tabs) and load grid (lg_tabs): rebuilt on every call.
// - grid (grid_tabs): the lists are uploaded only when epoch_tokens, the batch list or the replica list changed,
//   which leaves wva_grid_solve_device as the only call that can find them unchanged.  build_pair_tables (with the
//   per-(table, batch) constants) runs on every call: the tables are part of the evaluation.
// - sweep: builds into grid_tabs on every call; the upload leaves them keyed kUncached, so the grid's next call
//   uploads its own lists again.
template <class Fill>
int upload_tables(wva_handle* h, PairTables& pt, const std::vector<int>& pair, const std::vector<int>& len,
                  bool with_ls, Cols& c, Fill&& fill) {
    const int n = (int)pair.size();
    pt.epoch = kUncached;
    pt.key.clear();
    pt.o_pair = c.take(4 * (size_t)n);
    pt.o_off = c.take(8 * (size_t)n);
    pt.o_len = c.take(4 * (size_t)n);
    std::vector<char> host(c.bytes);
    char* p = host.data();
    long long entries = 0;
    pt.len_max = 1;
    for (int t = 0; t < n; ++t) {
        ((int*)(p + pt.o_pair))[t] = pair[t];
        ((long long*)(p + pt.o_off))[t] = entries;
        ((int*)(p + pt.o_len))[t] = len[t];
        entries += len[t];
        pt.len_max = std::max(pt.len_max, len[t]);
    }
    for (const Cols::Src& s : c.in) memcpy(p + s.off, s.src, s.bytes);
    fill(p);
    CK(pt.lists.ensure(c.bytes));
    // pageable source: cudaMemcpyAsync has consumed it by the time it returns
    CK(cudaMemcpyAsync(pt.lists.p, p, c.bytes, cudaMemcpyHostToDevice, h->stream));
    if (n) {
        CK(pt.tab.ensure(sizeof(double) * 4 * (size_t)entries));
        if (with_ls) CK(pt.ls.ensure(sizeof(float) * ((size_t)entries + n)));
    }
    pt.n = n;
    pt.with_ls = with_ls;
    return WVA_OK;
}

// build_pair_tables over the uploaded lists of fleet f's pairs; the grid passes its batch list and gets the
// per-(table, batch) constants in pb, and its n_zero step counters are zeroed (by one CTA when there is no table)
int build_tables(wva_handle* h, const DevFleet& f, const PairTables& pt, const int* batch = nullptr, int B = 0,
                 float4* pb = nullptr, unsigned* zero = nullptr, int n_zero = 0) {
    if (pt.n == 0 && n_zero == 0) return WVA_OK;
    build_pair_tables<<<std::max(pt.n, 1), 128, 0, h->stream>>>(f, pt.pair(), pt.off(), pt.len(), pt.n,
                                                                (double*)pt.tab.p, pt.with_ls ? (float*)pt.ls.p : nullptr,
                                                                batch, B, pb, zero, n_zero);
    h->launches++;
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- size path (K1) ---------------------------------------------------------
// one table per load pair (N entries), sorted by descending N
int prepare_size(wva_handle* h) {
    PairTables& pt = h->size_tabs;
    if (pt.holds(h->epoch_tokens)) return WVA_OK;
    const HostFleet& hf = h->hf;
    std::vector<int> pairs, Ns;
    int rc = sorted_pairs(h, hf, [&](int s, int a) { return hf.pair_class(s, a, true) == PAIR_LOAD; }, pairs, Ns);
    if (rc) return rc;
    Cols c(16);
    rc = upload_tables(h, pt, pairs, Ns, true, c, [](char*) {});
    if (rc) return rc;
    rc = build_tables(h, h->df, pt);
    if (rc) return rc;
    pt.epoch = h->epoch_tokens;
    return WVA_OK;
}

// Round-based K1 with speculative bisection trees: see the comment at the top of wva_size.cuh.
int size_depth_for(int n) {
    int d = n <= 2048 ? 5 : (n <= 8192 ? 4 : (n <= 40000 ? 3 : 2));
    if (const char* e = getenv("WVA_SIZE_DEPTH")) d = atoi(e);
    return std::min(std::max(d, 1), kSzMaxDepth);
}
// What the size drivers compute per candidate: CreateAllocation, its rateStar mode (the load grid) or its search
// mode (the SLO grid).
enum SizeMode { SIZE_FULL, SIZE_STAR, SIZE_SEARCH };
int run_size_rounds(wva_handle* h, const SizeArgs& sa, int n, SizeMode mode, const SearchCols& search) {
    const int D = size_depth_for(n);
    const size_t per_cand = 2 * ((size_t)(1 << D) - 1 + 2);  // two searches: a tree each, plus the two end points
    const size_t cap = per_cand * (size_t)n;                 // requests per round, worst case
    if (cap >= 0xffffffffull) return h->fail(WVA_ERR_UNSUPPORTED, "too many size candidates for one call (request slots are 32-bit)");
    const size_t n2 = 2 * (size_t)n;
    // state block
    Cols st(16);
    const size_t o_xmin = st.take(4 * n2), o_xmax = st.take(4 * n2), o_xs = st.take(4 * n2);
    const size_t o_sst = st.take(n2), o_inc = st.take(n2), o_iter = st.take(n2), o_ind = st.take(n2),
                 o_slot = st.take(4 * n2);
    const size_t o_phase = st.take(n), o_rmax = st.take(4 * (size_t)n), o_l2s0 = st.take(4 * (size_t)n),
                 o_l2sN = st.take(4 * (size_t)n), o_lsN = st.take(4 * (size_t)n), o_rstar = st.take(4 * (size_t)n),
                 o_cost = st.take(4 * (size_t)n), o_nrep = st.take(8 * (size_t)n), o_aslot = st.take(4 * (size_t)n);
    CK(h->d_sz_state.ensure(st.bytes));
    char* sp = (char*)h->d_sz_state.p;
    // request block
    Cols rq(16);
    const size_t r_id = rq.take(4 * cap), r_lam = rq.take(4 * cap), r_key = rq.take(cap), r_out = rq.take(16 * cap),
                 r_bail = rq.take(cap), r_cnt = rq.take(16);
    CK(h->d_sz_req.ensure(rq.bytes));
    char* rp = (char*)h->d_sz_req.p;
    // sort workspace
    const size_t chunks = (cap + kSortChunk - 1) / kSortChunk;
    const size_t max_items = (cap + 31) / 32 + chunks;
    Cols ws(16);
    const size_t w_order = ws.take(4 * cap), w_items = ws.take(8 * max_items), w_sorted = ws.take(8 * max_items),
                 w_cnt = ws.take(4 * (2 * kClasses + 8));
    CK(h->d_sz_sort.ensure(ws.bytes));
    char* wp = (char*)h->d_sz_sort.p;
    CK(h->sz_pin.ensure(64));

    Sz2Args g{};
    g.f = sa.f;
    g.cand_pair = sa.cand_pair;
    g.cand_N = sa.cand_N;
    g.n_cand = n;
    g.depth = D;
    g.tab = sa.tab;
    g.tab_off = sa.tab_off;
    g.ls = sa.ls;
    g.place = sa.place;
    g.xmin = (float*)(sp + o_xmin); g.xmax = (float*)(sp + o_xmax); g.xs = (float*)(sp + o_xs);
    g.sst = (uint8_t*)(sp + o_sst); g.inc = (uint8_t*)(sp + o_inc); g.iter = (uint8_t*)(sp + o_iter);
    g.ind = (int8_t*)(sp + o_ind); g.slot = (int*)(sp + o_slot);
    g.phase = (uint8_t*)(sp + o_phase);
    g.rmax = (float*)(sp + o_rmax); g.l2s0 = (float*)(sp + o_l2s0); g.l2sN = (float*)(sp + o_l2sN); g.lsN = (float*)(sp + o_lsN);
    g.rate_star = (float*)(sp + o_rstar); g.cost = (float*)(sp + o_cost);
    g.nrep = (long long*)(sp + o_nrep);
    g.aslot = (int*)(sp + o_aslot);
    g.req_id = (unsigned*)(rp + r_id); g.req_lam = (float*)(rp + r_lam); g.req_key = (uint8_t*)(rp + r_key);
    g.req_out = (float4*)(rp + r_out); g.req_bail = (uint8_t*)(rp + r_bail);
    g.n_req = (unsigned*)(rp + r_cnt); g.n_live = g.n_req + 1;
    g.ws.order = (unsigned*)(wp + w_order); g.ws.items = (unsigned long long*)(wp + w_items);
    g.ws.items_sorted = (unsigned long long*)(wp + w_sorted); g.ws.item_count = (unsigned*)(wp + w_cnt);
    g.cand = sa.cand;
    g.fb = sa.fb;
    g.search = search;

    const unsigned nb = (unsigned)((n + 255) / 256);
    const unsigned cks = (unsigned)chunks, items_blocks = (unsigned)((max_items + 255) / 256),
                   solve_blocks = (unsigned)((max_items * 32 + 255) / 256);
    if (mode == SIZE_SEARCH) sz2_init_search<<<nb, 256, 0, h->stream>>>(g);
    else sz2_init<<<nb, 256, 0, h->stream>>>(g);
    h->launches++;
    unsigned* pin = (unsigned*)h->sz_pin.p;
    // Rounds are enqueued in groups without looking at the device: every kernel of a round leaves at once when the
    // round has no requests, so over-launching costs microseconds while a host round trip per round costs more.
    // A search needs 1 + ceil(100 / D) rounds at most, then two Analyze rounds and the final consume.
    const int max_rounds = 1 + (100 + D - 1) / D + 4;
    const int group = 4;
    for (int round = 0; round < max_rounds; round += group) {
        for (int r = 0; r < group; ++r) {
            sz2_round_reset<<<3, 256, 0, h->stream>>>(g);
            if (mode == SIZE_STAR) sz2_advance_star<<<nb, 256, 0, h->stream>>>(g);
            else if (mode == SIZE_SEARCH) sz2_advance_search<<<nb, 256, 0, h->stream>>>(g);
            else sz2_advance<<<nb, 256, 0, h->stream>>>(g);
            sz2_sort_local<<<cks, kSortThreads, 0, h->stream>>>(g);
            ws_items_scan<<<1, 256, 0, h->stream>>>(g.ws);
            ws_items_scatter<<<items_blocks, 256, 0, h->stream>>>(g.ws);
            sz2_solve<<<solve_blocks, 256, 0, h->stream>>>(g);
            h->launches += 6;
        }
        // candidates still unfinished after the group's last advance decide whether another group is needed
        CK(cudaMemcpyAsync(pin, g.n_live, sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        if (*pin == 0) break;
    }
    CK(cudaGetLastError());
    return WVA_OK;
}

// CreateAllocation for the load candidates g lists (g.cand_pair .. g.place set, batch sizes at most Nmax), up to
// rateStar in SIZE_STAR mode, or one search each in SIZE_SEARCH mode (with `search`): the warp-per-candidate kernel
// or the rounds, timed as the call's kernel, then the stored-vector fallback.
int enqueue_candidates(wva_handle* h, SizeArgs& g, int Nmax, SizeMode mode = SIZE_FULL, const SearchCols& search = {}) {
    const int n = g.n_cand;
    FbRun fb;
    const int rc = prepare_fallback(h, 0, n, n ? Nmax : 0, fb);
    if (rc) return rc;
    g.fb = fb.list;
    CK(cudaEventRecord(h->ev_k0, h->stream));
    int small_max = 1024;  // up to here a warp per candidate beats rounds (the GPU is mostly empty either way)
    if (const char* e = getenv("WVA_SIZE_SMALL_MAX")) small_max = atoi(e);
    if (n > 0 && n <= small_max) {
        const unsigned blocks = (unsigned)((n + 3) / 4);
        if (mode == SIZE_STAR) size_warp_star<<<blocks, 128, 0, h->stream>>>(g);
        else if (mode == SIZE_SEARCH) size_warp_search<<<blocks, 128, 0, h->stream>>>(SearchArgs{g, search});
        else size_warp_kernel<<<blocks, 128, 0, h->stream>>>(g);
        h->launches++;
    } else if (n > 0) {
        const int rc = run_size_rounds(h, g, n, mode, search);
        if (rc) return rc;
    }
    CK(cudaEventRecord(h->ev_k1, h->stream));
    if (n > 0 && mode == SIZE_SEARCH) launch_fallback(h, size_fallback_search, SearchArgs{g, search}, fb);
    else if (n > 0) launch_fallback(h, mode == SIZE_STAR ? size_fallback_star : size_fallback, g, fb);
    CK(cudaGetLastError());
    return WVA_OK;
}

// The size drivers' arguments for fleet f: one candidate per table of pt, written into cand by pair id.
SizeArgs size_args(const DevFleet& f, const PairTables& pt, const AllocCols& cand) {
    SizeArgs g{};
    g.f = f;
    g.cand_pair = pt.pair();
    g.cand_N = pt.len();
    g.n_cand = pt.n;
    g.tab = (const double*)pt.tab.p;
    g.tab_off = pt.off();
    g.ls = (const float*)pt.ls.p;
    g.place = CandPlace{nullptr, nullptr};
    g.cand = cand;
    return g;
}

// Enqueue analyze (+ unlimited solve). cand/winner columns are device pointers.
int enqueue_size(wva_handle* h, const AllocCols& cand, const AllocCols* winners) {
    int rc = prepare_size(h);
    if (rc) return rc;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    const HostFleet& hf = h->hf;
    launch_records(h, (long long)hf.S * hf.A, trivial_kernel, h->df, cand, (const int*)nullptr, 1);
    const PairTables& pt = h->size_tabs;
    SizeArgs g = size_args(h->df, pt, cand);
    rc = enqueue_candidates(h, g, pt.len_max);
    if (rc) return rc;
    if (winners && hf.S > 0) {
        unlimited_kernel<<<(hf.S + 127) / 128, 128, 0, h->stream>>>(h->df, cand, *winners);
        h->launches++;
    }
    CK(cudaGetLastError());
    return WVA_OK;
}

int finish_timing(wva_handle* h) {
    CK(cudaEventRecord(h->ev_d1, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    cudaEventElapsedTime(&h->last_kernel_ms, h->ev_k0, h->ev_k1);
    cudaEventElapsedTime(&h->last_device_ms, h->ev_d0, h->ev_d1);
    return WVA_OK;
}

// What a call with host results places on the device and copies back.  Every call has a winner block ([S], [L*S]
// for the load grid); the size path also writes a candidate block ([S*A], [S*A*B] for the size grid, [L*S*A] for
// the load grid).
struct HostCall {
    size_t n_cand;                  // records of the candidate block the work writes (0: none)
    bool copy_cand, copy_win;       // which blocks come back to the host
    const Cols* extra = nullptr;    // further device columns copied straight to their destinations ...
    const void* extra_dev = nullptr;  // ... from this buffer
    size_t win_blocks = 1;          // winner blocks of S records
    // set by run_host: the block layouts and their host copies in out_stage (NULL when not copied)
    Block bc{}, bw{};
    const char *cand_host = nullptr, *win_host = nullptr;
};

// The shared end of every call with host results, in stream order: place the blocks on the device, record
// ev_d0, enqueue the work, copy the wanted blocks and the control ints into out_stage and then c.extra,
// synchronise once and check the fallback's status words.  enqueue(dc, dw) enqueues the kernels into the device
// blocks.
template <class Enqueue>
int run_host(wva_handle* h, HostCall& c, Enqueue&& enqueue) {
    const HostFleet& hf = h->hf;
    c.bc = block_layout(c.n_cand);
    c.bw = block_layout((size_t)hf.S * c.win_blocks);
    if (c.n_cand) CK(h->d_cand_block.ensure(c.bc.bytes + 16));
    CK(h->d_win_block.ensure(c.bw.bytes + 16));
    const AllocCols dc = c.n_cand ? block_cols(h->d_cand_block.p, c.bc) : AllocCols{};
    const AllocCols dw = block_cols(h->d_win_block.p, c.bw);
    CK(cudaEventRecord(h->ev_d0, h->stream));
    int rc = enqueue(dc, dw);
    if (rc) return rc;
    Cols stage(256);
    const size_t o_cand = stage.take(c.copy_cand ? c.bc.bytes : 0), o_win = stage.take(c.copy_win ? c.bw.bytes : 0),
                 o_ctrl = stage.take(CTRL_INTS * sizeof(int));
    CK(h->out_stage.ensure(stage.bytes));
    char* hs = (char*)h->out_stage.p;
    if (c.copy_cand) {
        CK(cudaMemcpyAsync(hs + o_cand, h->d_cand_block.p, c.bc.bytes, cudaMemcpyDeviceToHost, h->stream));
        c.cand_host = hs + o_cand;
    }
    if (c.copy_win) {
        CK(cudaMemcpyAsync(hs + o_win, h->d_win_block.p, c.bw.bytes, cudaMemcpyDeviceToHost, h->stream));
        c.win_host = hs + o_win;
    }
    const int* ctrl = (const int*)(hs + o_ctrl);
    CK(cudaMemcpyAsync(hs + o_ctrl, h->d_ctrl.p, CTRL_INTS * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    if (c.extra) CK(c.extra->copy_back(c.extra_dev, h->stream));
    rc = finish_timing(h);
    if (rc) return rc;
    if (ctrl[CTRL_FB_STATUS] != 0)
        return h->fail(WVA_ERR_UNSUPPORTED, "input outside the supported numeric domain (rescale loop does not terminate)");
    if (ctrl[CTRL_FB_OVERFLOW] != 0)
        return h->fail(WVA_ERR_UNSUPPORTED, "too many entries need the stored-vector fallback");
    return WVA_OK;
}

// resident analyze/solve with host outputs
int run_size_host(wva_handle* h, wva_allocs* candidates, wva_allocs* winners) {
    if (!h->resident) return h->fail(WVA_ERR_STATE, "no resident fleet (call wva_upload first)");
    HostCall c{(size_t)h->hf.S * h->hf.A, candidates != nullptr, winners != nullptr};
    const int rc = run_host(h, c, [&](const AllocCols& dc, const AllocCols& dw) {
        return enqueue_size(h, dc, winners ? &dw : nullptr);
    });
    if (rc) return rc;
    scatter_block(c.cand_host, c.bc, candidates);
    scatter_block(c.win_host, c.bw, winners);
    return WVA_OK;
}

// The entry of the calls over L rows of a fleet with L candidate and L winner blocks (the load, SLO, workload and
// profile grids, the workload and profile traces), named `name` in wva_last_error: the argument checks, the upload,
// then enqueue(dc, dw) under run_host and both blocks back to the caller.  null_rows is the call's refusal when some
// row list it needs is NULL (it applies when S * L > 0), or NULL; with row_entries the L * M * A entries of a
// wva_profile_rows list are bounded as well.  A trace's rows are ticks, a grid's levels.  A call with outputs beyond
// the two blocks (the price threshold grid and trace) passes `more`.
struct LevelMore {
    std::function<int(HostCall&)> place;        // after the upload, before any launch: refuse, or set c.extra
    std::function<int(const HostCall&)> check;  // after the sync, before the blocks reach the caller: refuse
};
template <class Enqueue>
int run_levels(wva_handle* h, const wva_fleet* fleet, int32_t L, const char* name, const char* null_rows,
               bool row_entries, wva_allocs* candidates, wva_allocs* winners, Enqueue&& enqueue,
               const LevelMore& more = LevelMore{}) {
    if (!h || !winners) return WVA_ERR_BAD_ARG;
    if (L < 0) return h->fail(WVA_ERR_BAD_ARG, strstr(name, "trace") ? "negative tick count" : "negative level count");
    if (!fleet) return h->fail(WVA_ERR_BAD_ARG, "fleet is NULL");
    if ((long long)fleet->n_servers * L > 0 && null_rows) return h->fail(WVA_ERR_BAD_ARG, null_rows);
    const long long n_cand = (long long)fleet->n_servers * fleet->n_acc * L;
    if (n_cand >= (1ll << 31) || (row_entries && (long long)L * fleet->n_models * fleet->n_acc >= (1ll << 31))) {
        const std::string what = std::string(name) + " too large for one call (>= 2^31 candidates" +
                                 (row_entries ? " or row entries)" : ")");
        return h->fail(WVA_ERR_UNSUPPORTED, what.c_str());
    }
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    HostCall c{(size_t)n_cand, candidates != nullptr, true};
    c.win_blocks = (size_t)L;
    if (more.place && (rc = more.place(c))) return rc;
    rc = run_host(h, c, enqueue);
    // no single solution to summarise (upload_fleet cleared last_kind)
    if (rc) return rc;
    if (more.check && (rc = more.check(c))) return rc;
    scatter_block(c.cand_host, c.bc, candidates);
    scatter_block(c.win_host, c.bw, winners);
    return WVA_OK;
}

// ---- size grid: CreateAllocation at every listed batch size --------------------------------------
// The load pairs x the batch list, sorted by descending N (stable: pair order, then list order), with one
// Bmax-long table per pair that the pair's candidates share.  Enqueues the nil / zero-load candidates,
// CreateAllocation for the load candidates, then values and the per-server winners.  cand ([S*A*B]) and winners
// ([S]) are device columns.
int enqueue_size_grid(wva_handle* h, int B, const int32_t* batch, const AllocCols& cand, const AllocCols& winners) {
    const HostFleet& hf = h->hf;
    PairTables& pt = h->sg_tabs;
    int Bmax = 1;
    for (int i = 0; i < B; ++i) Bmax = std::max(Bmax, batch[i]);
    std::vector<int> tab_pair;
    for (int s = 0; s < hf.S; ++s)
        for (int a = 0; a < hf.A; ++a)
            if (hf.pair_class(s, a, true) == PAIR_LOAD) tab_pair.push_back(s * hf.A + a);
    const int n_tab = (int)tab_pair.size();
    if ((long long)n_tab * Bmax > 0xffffffffll) return h->fail(WVA_ERR_UNSUPPORTED, "size-grid tables above 2^32 entries");
    if (n_tab > 0 && B > 0 && !hf.queue_fits(Bmax))
        return h->fail(WVA_ERR_UNSUPPORTED,
                       "queue model of 2^31 states or more (batch size x (1 + max_queue_to_batch_ratio))");
    const int n = n_tab * B;  // <= S * A * B < 2^31 (checked by the caller)
    std::vector<int> order(n);  // candidate t * B + bi of table t
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return batch[x % B] > batch[y % B]; });
    Cols c(16);
    const size_t o_pair = c.take(4 * (size_t)n), o_N = c.take(4 * (size_t)n), o_rec = c.take(4 * (size_t)n),
                 o_idx = c.take(4 * (size_t)n), o_off = c.take(8 * (size_t)n), o_bl = c.put(batch, 4 * (size_t)B);
    int rc = upload_tables(h, pt, tab_pair, std::vector<int>(n_tab, Bmax), true, c, [&](char* p) {
        for (int j = 0; j < n; ++j) {
            const int t = order[j] / B, bi = order[j] % B;
            ((int*)(p + o_pair))[j] = tab_pair[t];
            ((int*)(p + o_N))[j] = batch[bi];
            ((int*)(p + o_rec))[j] = tab_pair[t] * B + bi;
            ((int*)(p + o_idx))[j] = t;
            ((long long*)(p + o_off))[j] = (long long)t * Bmax;
        }
    });
    if (rc) return rc;
    rc = build_tables(h, h->df, pt);
    if (rc) return rc;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    const char* d = (const char*)pt.lists.p;
    const int* d_batch = (const int*)(d + o_bl);
    launch_records(h, (long long)hf.S * hf.A * B, trivial_kernel, h->df, cand, d_batch, B);
    SizeArgs g = size_args(h->df, pt, cand);
    g.cand_pair = (const int*)(d + o_pair);
    g.cand_N = (const int*)(d + o_N);
    g.n_cand = n;
    g.tab_off = (const long long*)(d + o_off);
    g.place = CandPlace{(const int*)(d + o_idx), (const int*)(d + o_rec)};
    rc = enqueue_candidates(h, g, Bmax);
    if (rc) return rc;
    if (hf.S > 0) {
        size_grid_finalize<<<(unsigned)((hf.S + 3) / 4), 128, 0, h->stream>>>(h->df, cand, d_batch, B, winners);
        h->launches++;
    }
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- load grid: CreateAllocation and the unlimited winner at every listed load level -------------------------
// Phase 1 sizes each candidate once: the pairs that pass the gates and are a load somewhere in the caller's
// rates, sorted by descending N with one N-entry table each, run through the size drivers in rateStar mode.  The
// load grid, the load intervals and the workload grid share it (and lg_tabs / d_lg_star, which all rebuild on every
// call).  Each passes the fleet it sizes: the resident one, or the workload grid's key fleet.
//
// prepare_load_star uploads the candidate lists of fleet hf with the caller's columns (laid out in c, written by
// fill; `pairs` holds the candidates' pair ids by the time fill runs).  pin, when given (a trace's trace_pinned
// flags), keeps keepAccelerator on the pinned servers only.  enqueue_load_star then builds the tables
// for the device image f of the same fleet and sizes fallback list 1 for the caller's tail (prepare_tail, which the
// SLO grid shares), and enqueues phase 1.
struct LoadStar {
    AllocCols star{};    // rateStar mode's records by pair id: feasible and max_rate = rateStar
    FbRun fb2{};         // the tail's fallback list
    SizeArgs g{};        // phase 1's fleet, candidates and tables
};
template <class Fill>
int prepare_load_star(wva_handle* h, const HostFleet& hf, const std::vector<char>& loaded, std::vector<int>& pairs,
                      Cols& c, Fill&& fill, const uint8_t* pin = nullptr) {
    std::vector<int> Ns;
    int rc = sorted_pairs(
        h, hf,
        [&](int s, int a) { return loaded[s] && hf.pair_class(s, a, !pin || pin[s], 1.0f) == PAIR_LOAD; }, pairs,
        Ns);
    if (rc) return rc;
    return upload_tables(h, h->lg_tabs, pairs, Ns, true, c, fill);
}
// Builds lg_tabs' tables for fleet f and sizes the tail's fallback list (list 1, up to fb2_cap entries) before
// phase 1 is enqueued (which sizes the scratch for the same len_max).  Needs ensure_ctrl.
int prepare_tail(wva_handle* h, const DevFleet& f, long long fb2_cap, FbRun& fb2) {
    const PairTables& pt = h->lg_tabs;
    const int rc = build_tables(h, f, pt);
    if (rc) return rc;
    return prepare_fallback(h, 1, (int)std::min<long long>(fb2_cap, 1 << 22), pt.n ? pt.len_max : 0, fb2);
}
int enqueue_load_star(wva_handle* h, const HostFleet& hf, const DevFleet& f, long long fb2_cap, LoadStar& ls) {
    const PairTables& pt = h->lg_tabs;
    const size_t n_pairs = (size_t)hf.S * hf.A;
    CK(h->d_lg_star.ensure(5 * n_pairs + 16));
    ls.star = AllocCols{};
    ls.star.max_rate = (float*)h->d_lg_star.p;
    ls.star.feasible = (uint8_t*)h->d_lg_star.p + 4 * n_pairs;
    const int rc = prepare_tail(h, f, fb2_cap, ls.fb2);
    if (rc) return rc;
    ls.g = size_args(f, pt, ls.star);
    return enqueue_candidates(h, ls.g, pt.len_max, SIZE_STAR);
}

// The winners of an L-block call: per block the unlimited winner (unlimited_kernel), or with `trace` the workload
// trace's tick chain (trace_kernel), in which block l's winners are block l + 1's current allocation.
void enqueue_level_winners(wva_handle* h, const AllocCols& cand, const AllocCols& winners, int L, bool trace) {
    const int S = h->hf.S;
    if (S <= 0 || L <= 0) return;
    if (trace)
        trace_kernel<<<(unsigned)((S + 127) / 128), 128, 0, h->stream>>>(h->df, cand, winners, L);
    else
        unlimited_kernel<<<dim3((unsigned)((S + 127) / 128), (unsigned)std::min(L, 65535)), 128, 0, h->stream>>>(
            h->df, cand, winners, L);
    h->launches++;
}
// A tail's fleet f, and its candidates and tables: those of pt, one per table.
template <class Args>
void set_tables(Args& g, const DevFleet& f, const PairTables& pt) {
    g.f = f;
    g.cand_pair = pt.pair();
    g.cand_N = pt.len();
    g.tab_off = pt.off();
    g.tab = (const double*)pt.tab.p;
    g.n_cand = pt.n;
}
// The tail's view of phase 1: fleet, candidates, tables and rateStar records (the level list is the caller's).
LoadArgs load_args(wva_handle* h, const LoadStar& ls) {
    LoadArgs la{};
    set_tables(la, ls.g.f, h->lg_tabs);
    la.star_ok = ls.star.feasible;
    la.rate_star = ls.star.max_rate;
    la.fb = ls.fb2.list;
    return la;
}

// One call's [L*S] lists of the server columns that a grid or trace replaces by row: arrival_rpm, in / out tokens
// and the ITL / TTFT / TPS targets.  The put_* calls put the lists the call reads into its upload image c, a NULL
// list tiled from the resident column (the calls that refuse NULL lists do so in run_levels).  After the upload, a
// list's dev() is its device pointer (NULL: not put) and load() the records' load rows.  The tiled lists live
// here, so a RowLists outlives the upload.
struct RowLists {
    template <class T>
    struct List {
        const T* host = nullptr;  // the caller's list or own
        size_t off = 0;
        bool placed = false;
        std::vector<T> own;
        const T* dev(const char* d) const { return placed ? (const T*)(d + off) : nullptr; }
    };
    const HostFleet& hf;
    int L;
    Cols& c;
    List<float> rpm, itl, ttft, tps;
    List<int32_t> in, out;

    void put_rpm(const float* r) { put(rpm, r, hf.srv_arrival_rpm); }
    void put_tokens(const int32_t* i, const int32_t* o) {
        put(in, i, hf.srv_in_tokens);
        put(out, o, hf.srv_out_tokens);
    }
    void put_targets(const float* i, const float* t, const float* p) {
        put(itl, i, hf.srv_slo_itl);
        put(ttft, t, hf.srv_slo_ttft);
        put(tps, p, hf.srv_slo_tps);
    }
    LoadRows load(const char* d) const { return LoadRows{rpm.dev(d), in.dev(d), out.dev(d)}; }

  private:
    template <class T>
    void put(List<T>& r, const T* list, const std::vector<T>& col) {
        const size_t S = col.size();
        if (!list) {
            r.own.resize((size_t)L * S);
            for (int l = 0; l < L; ++l) std::copy(col.begin(), col.end(), r.own.begin() + (size_t)l * S);
            list = r.own.data();
        }
        r.host = list;
        r.off = c.put(list, sizeof(T) * (size_t)L * S);
        r.placed = true;
    }
};

// Phase 2 (load_kernel, load_fallback) is the tail per (candidate, level).  rpm [L*S] is the caller's level list;
// cand ([L*S*A]) and winners ([L*S]) are device columns.
int enqueue_load_grid(wva_handle* h, int L, const float* rpm, const AllocCols& cand, const AllocCols& winners) {
    const HostFleet& hf = h->hf;
    const int S = hf.S, A = hf.A;
    std::vector<char> loaded(S, 0);  // server s is a load at some level (NaN and +Inf included)
    for (int l = 0; l < L; ++l)
        for (int s = 0; s < S; ++s) loaded[s] |= !(rpm[(size_t)l * S + s] < 0.0f) && rpm[(size_t)l * S + s] != 0.0f;
    std::vector<int> pairs;
    Cols c(16);
    RowLists lists{hf, L, c};
    lists.put_rpm(rpm);
    int rc = prepare_load_star(h, hf, loaded, pairs, c, [](char*) {});
    if (rc) return rc;
    const int n = (int)pairs.size();
    const long long n_items = (long long)n * L;
    const char* d = (const char*)h->lg_tabs.lists.p;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    launch_records(h, (long long)S * A * L, trivial_kernel, h->df, cand, lists.load(d), L);
    LoadStar ls;
    rc = enqueue_load_star(h, hf, h->df, n_items, ls);
    if (rc) return rc;
    if (n > 0 && L > 0) {
        LoadArgs la = load_args(h, ls);
        la.level_rpm = lists.rpm.dev(d);
        la.L = L;
        la.counter = (unsigned*)h->d_ctrl.p + CTRL_COUNTER;
        la.cand = cand;
        rc = launch_tail(h, load_kernel, load_fallback, la, (n_items + 31) / 32, ls.fb2);
        if (rc) return rc;
    }
    enqueue_level_winners(h, cand, winners, L, false);
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- token keys: the workload calls' distinct (server, in_tokens, out_tokens) rows (DESIGN.md §3.12) -----------
// Which lengths of WVA_FLEET_COLUMNS are per server.
#define WVA_PER_SERVER_A 0
#define WVA_PER_SERVER_T 0
#define WVA_PER_SERVER_MA 0
#define WVA_PER_SERVER_S 1
// ... per (model, accelerator): a key fleet of the profile grid has its own (own_ma).
#define WVA_PER_MODEL_A 0
#define WVA_PER_MODEL_T 0
#define WVA_PER_MODEL_MA 1
#define WVA_PER_MODEL_S 0

// The fleet the workload grid sizes (DESIGN.md §3.12): row k is server srv[k] of the resident fleet at the key's
// tokens, with a positive rate (phase 1 reads no rate; the tail reads the level's).  The A, T and M columns are the
// resident fleet's.  On the device the server columns lie in an upload image of the caller's (place), and
// view() points a copy of the resident DevFleet at them, so the resident arena is never written.  The profile grid
// also gives the key fleet its own models (own_ma): M and the perf_* columns are then the key fleet's.
struct KeyFleet {
    HostFleet hf;
    bool own_ma = false;
    struct {
#define KEY_OFFSET(abi, name, type, len) size_t name = 0;
        WVA_FLEET_COLUMNS(KEY_OFFSET)
#undef KEY_OFFSET
    } off;
    KeyFleet(const HostFleet& fleet, const std::vector<int>& srv, const std::vector<int>& in,
             const std::vector<int>& out)
        : hf(fleet) {
        const size_t K = srv.size();
        hf.S = (int)K;
#define KEY_GATHER(abi, name, type, len)                                     \
    if (WVA_PER_SERVER_##len) {                                              \
        hf.name.resize(K);                                                   \
        for (size_t k = 0; k < K; ++k) hf.name[k] = fleet.name[srv[k]];      \
    }
        WVA_FLEET_COLUMNS(KEY_GATHER)
#undef KEY_GATHER
        std::fill(hf.srv_arrival_rpm.begin(), hf.srv_arrival_rpm.end(), 1.0f);
        hf.srv_in_tokens = in;
        hf.srv_out_tokens = out;
    }
    void place(Cols& c) {
#define KEY_PLACE(abi, name, type, len)                            \
    if (WVA_PER_SERVER_##len || (own_ma && WVA_PER_MODEL_##len)) \
        off.name = c.put(hf.name.data(), sizeof(type) * hf.name.size());
        WVA_FLEET_COLUMNS(KEY_PLACE)
#undef KEY_PLACE
    }
    DevFleet view(DevFleet f, const char* d) const {
        f.S = hf.S;
        if (own_ma) f.M = hf.M;
#define KEY_VIEW(abi, name, type, len) \
    if (WVA_PER_SERVER_##len || (own_ma && WVA_PER_MODEL_##len)) f.name = (const type*)(d + off.name);
        WVA_FLEET_COLUMNS(KEY_VIEW)
#undef KEY_VIEW
        return f;
    }
};

// [L*S] lists of the ITL, TTFT and TPS targets by row: the SLO margins' (DESIGN.md §3.24), all three given.
struct TargetRows {
    const float* itl;
    const float* ttft;
    const float* tps;
};

// A key of load_groups: (in << 32) | out, then the bits of (ITL << 32) | TTFT and of TPS (0 without target rows).
using LoadKey = std::array<uint64_t, 3>;
using LoadUses = std::vector<std::pair<LoadKey, int>>;

// The levels at which server s is a load under the rows rpm / in / out [L*S] (rate not negative and not 0, NaN and
// +Inf included; in_tokens >= 0; out_tokens >= 1), as (key, level) in `uses`, sorted, the key being the level's
// tokens and, with tg, its targets' bits; then group(in, out, u0, u1) for each key in ascending order, whose levels
// are uses[u0 .. u1), ascending.  Without tg the keys are the (in, out) pairs.
template <class Group>
void load_groups(int L, int S, int s, const float* rpm, const int32_t* in, const int32_t* out, LoadUses& uses,
                 Group&& group, const TargetRows* tg = nullptr) {
    const auto bits = [](float x) {
        uint32_t u;
        memcpy(&u, &x, 4);
        return (uint64_t)u;
    };
    uses.clear();
    for (int l = 0; l < L; ++l) {
        const size_t i = (size_t)l * S + s;
        if (!(rpm[i] < 0.0f) && rpm[i] != 0.0f && in[i] >= 0 && out[i] >= 1) {
            LoadKey k{(uint64_t)(uint32_t)in[i] << 32 | (uint32_t)out[i], 0, 0};
            if (tg) k = {k[0], bits(tg->itl[i]) << 32 | bits(tg->ttft[i]), bits(tg->tps[i])};
            uses.emplace_back(k, l);
        }
    }
    std::sort(uses.begin(), uses.end());
    for (size_t u0 = 0, u1; u0 < uses.size(); u0 = u1) {
        for (u1 = u0; u1 < uses.size() && uses[u1].first == uses[u0].first;) ++u1;
        group((int)(uses[u0].first[0] >> 32), (int)(uint32_t)uses[u0].first[0], u0, u1);
    }
}

// Key rows (server, in_tokens, out_tokens) with their levels: row k's are lev[lev_off[k] .. lev_off[k + 1]).  On
// the device the workload grid's tail reads the servers, the level lists and each candidate's first item, which
// lie in the call's upload image (place, write) and which args() hands to a WorkloadArgs.
struct TokenKeys {
    std::vector<int> srv, in, out, lev_off{0}, lev;
    size_t o_srv = 0, o_loff = 0, o_lev = 0, o_item = 0;
    int n_items = 0;  // set by write
    void add(int s, int ki, int ko) {
        srv.push_back(s);
        in.push_back(ki);
        out.push_back(ko);
        lev_off.push_back(lev_off.back());
    }
    void add_level(int l) {
        lev.push_back(l);
        lev_off.back()++;
    }
    // the key rows, and room for the item offsets of up to n_cand candidates
    void place(Cols& c, size_t n_cand) {
        o_srv = c.put(srv.data(), 4 * srv.size());
        o_loff = c.put(lev_off.data(), 4 * lev_off.size());
        o_lev = c.put(lev.data(), 4 * lev.size());
        o_item = c.take(4 * (n_cand + 1));
    }
    // candidate j's items: one per level of its key row pairs[j] / A
    void write(char* p, const std::vector<int>& pairs, int A) {
        int* item = (int*)(p + o_item);
        item[0] = 0;
        for (size_t j = 0; j < pairs.size(); ++j) {
            const int k = pairs[j] / A;
            item[j + 1] = item[j] + lev_off[k + 1] - lev_off[k];
        }
        n_items = item[pairs.size()];
    }
    // the tail's lists uploaded at d, for levels of S servers
    WorkloadArgs args(const char* d, int S) const {
        WorkloadArgs g{};
        g.key_srv = (const int*)(d + o_srv);
        g.lev_off = (const int*)(d + o_loff);
        g.lev = (const int*)(d + o_lev);
        g.item_off = (const int*)(d + o_item);
        g.S = S;
        g.n_items = n_items;
        return g;
    }
};
// The workload grid's keys (DESIGN.md §3.12) of the rows rpm / in / out into tk: per server, its distinct (in, out)
// under load, ascending.  Returns their key fleet, which with pin (a trace's trace_pinned flags) keeps
// keepAccelerator on the pinned servers only, so that phase 1 sizes their current accelerator alone.  With tg (the SLO
// margins, DESIGN.md §3.24) the keys are per server its distinct (in, out, target bits), and the key fleet's srv_slo_*
// columns hold each key's targets.
KeyFleet workload_keys(const HostFleet& hf, int L, const float* rpm, const int32_t* in, const int32_t* out,
                       const uint8_t* pin, TokenKeys& tk, const TargetRows* tg = nullptr) {
    LoadUses uses;
    for (int s = 0; s < hf.S; ++s)
        load_groups(
            L, hf.S, s, rpm, in, out, uses,
            [&](int ki, int ko, size_t u0, size_t u1) {
                tk.add(s, ki, ko);
                for (size_t u = u0; u < u1; ++u) tk.add_level(uses[u].second);
            },
            tg);
    KeyFleet kf(hf, tk.srv, tk.in, tk.out);
    if (pin)
        for (size_t k = 0; k < tk.srv.size(); ++k) kf.hf.srv_keep_acc[k] = pin[tk.srv[k]];
    if (tg)
        for (size_t k = 0; k < tk.srv.size(); ++k) {
            const size_t i = (size_t)tk.lev[tk.lev_off[k]] * hf.S + tk.srv[k];  // the key's first row
            kf.hf.srv_slo_itl[k] = tg->itl[i];
            kf.hf.srv_slo_ttft[k] = tg->ttft[i];
            kf.hf.srv_slo_tps[k] = tg->tps[i];
        }
    return kf;
}

// The rows of a wva_profile_rows list as the profile grid and the profile trace size them.  Per (m, a) the host ranks
// the distinct present rows that the levels use (elsewhere no pair of m is a load); key-model (m, j) = moff[m] + j
// holds the j-th distinct row of (m, a) at every accelerator a that has one, so a key fleet's tables stay within
// L * M * A entries.  The caller's row lists travel in the call's upload image (place), and set_rows points a
// ProfileArgs at them.
struct ProfileRanks {
    using Row = std::array<uint32_t, 6>;  // bits of alpha, beta, gamma, delta; max_batch, at_tokens
    const void* lists[9];                 // column c: the caller's row list (bit c of per_level) or NULL
    unsigned per_level = 0;
    bool perf_rows = false;               // some perf column is a row list
    int L, A;
    size_t MA;
    // the distinct present rows of (m, a) = k: row_v[row_off[k] .. row_off[k + 1]), ascending; rank [L*M*A] is row
    // (l, k)'s index among them (-1: absent), built only when perf_rows
    std::vector<Row> row_v;
    std::vector<int> row_off, rank;
    std::vector<int> moff;  // [M + 1]: key-model (m, j) = moff[m] + j, j < the most distinct rows of m at any a
    size_t o_list[9] = {};

    ProfileRanks(const HostFleet& hf, int L_, const wva_profile_rows& rows)
        : lists{rows.acc_cost,  rows.perf_present,   rows.perf_alpha,     rows.perf_beta,     rows.perf_gamma,
                rows.perf_delta, rows.perf_acc_count, rows.perf_max_batch, rows.perf_at_tokens},
          L(L_), A(hf.A), MA((size_t)hf.M * hf.A), row_off(MA + 1, 0), moff(hf.M + 1, 0) {
        for (int c = 0; c < 9; ++c) per_level |= lists[c] ? 1u << c : 0u;
        perf_rows = (per_level >> 1) != 0;
        // column c of row l at entry k
        auto at = [&](const auto* list, const auto& own, int l, size_t k) { return list ? list[l * MA + k] : own[k]; };
        auto bits = [](float x) {
            uint32_t u;
            memcpy(&u, &x, 4);
            return u;
        };
        auto row_of = [&](int l, size_t k) {
            return Row{bits(at(rows.perf_alpha, hf.perf_alpha, l, k)), bits(at(rows.perf_beta, hf.perf_beta, l, k)),
                       bits(at(rows.perf_gamma, hf.perf_gamma, l, k)), bits(at(rows.perf_delta, hf.perf_delta, l, k)),
                       (uint32_t)at(rows.perf_max_batch, hf.perf_max_batch, l, k),
                       (uint32_t)at(rows.perf_at_tokens, hf.perf_at_tokens, l, k)};
        };
        if (perf_rows) {
            rank.assign((size_t)L * MA, -1);
            std::vector<std::pair<Row, int>> uses;
            for (size_t k = 0; k < MA; ++k) {
                uses.clear();
                for (int l = 0; l < L; ++l)
                    if (at(rows.perf_present, hf.perf_present, l, k)) uses.emplace_back(row_of(l, k), l);
                std::sort(uses.begin(), uses.end());
                for (size_t u = 0; u < uses.size(); ++u) {
                    if (u == 0 || uses[u].first != uses[u - 1].first) row_v.push_back(uses[u].first);
                    rank[(size_t)uses[u].second * MA + k] = (int)row_v.size() - 1 - row_off[k];
                }
                row_off[k + 1] = (int)row_v.size();
            }
        } else {
            for (size_t k = 0; k < MA; ++k) {
                if (L > 0 && hf.perf_present[k]) row_v.push_back(row_of(0, k));
                row_off[k + 1] = (int)row_v.size();
            }
        }
        for (int m = 0; m < hf.M; ++m) {
            int J = 0;
            for (int a = 0; a < A; ++a) J = std::max(J, row_off[(size_t)m * A + a + 1] - row_off[(size_t)m * A + a]);
            moff[m + 1] = moff[m] + J;
        }
    }
    // row (l, k)'s index among the distinct rows of k, -1 where (m, a) is absent at row l
    int rank_at(int l, size_t k) const {
        if (perf_rows) return rank[(size_t)l * MA + k];
        return row_off[k + 1] > row_off[k] ? 0 : -1;
    }
    // What a load pair's sizing reads of row j of k = (m, a): ((alpha, beta), (gamma, delta), N), N being the
    // server's batch size max_batch when positive and the row's AtTokens rule at out_tokens out otherwise.
    std::array<uint64_t, 3> sizing_key(size_t k, int j, int max_batch, int out) const {
        const Row& r = row_v[row_off[k] + j];
        const long long t = (long long)(int32_t)r[4] * (int32_t)r[5] / out;
        const long long N = max_batch > 0 ? max_batch : std::max<long long>(t, 1);
        return {(uint64_t)r[0] << 32 | r[1], (uint64_t)r[2] << 32 | r[3], (uint64_t)N};
    }
    // the key fleet's models: M and the perf columns of the key-models (kh starts as a copy of the fleet)
    void fill(HostFleet& kh) const {
        kh.M = moff.back();
        const size_t KMA = (size_t)kh.M * A;
        kh.perf_present.assign(KMA, 0);
        kh.perf_acc_count.assign(KMA, 1);
        for (auto* col : {&kh.perf_alpha, &kh.perf_beta, &kh.perf_gamma, &kh.perf_delta}) col->assign(KMA, 0.0f);
        kh.perf_max_batch.assign(KMA, 0);
        kh.perf_at_tokens.assign(KMA, 0);
        for (size_t m = 0; m + 1 < moff.size(); ++m)
            for (int a = 0; a < A; ++a) {
                const size_t k = m * A + a;
                for (int j = 0; j < row_off[k + 1] - row_off[k]; ++j) {
                    const Row& r = row_v[row_off[k] + j];
                    const size_t q = (size_t)(moff[m] + j) * A + a;
                    kh.perf_present[q] = 1;
                    memcpy(&kh.perf_alpha[q], &r[0], 4);
                    memcpy(&kh.perf_beta[q], &r[1], 4);
                    memcpy(&kh.perf_gamma[q], &r[2], 4);
                    memcpy(&kh.perf_delta[q], &r[3], 4);
                    kh.perf_max_batch[q] = (int32_t)r[4];
                    kh.perf_at_tokens[q] = (int32_t)r[5];
                }
            }
    }
    size_t list_bytes(int c) const {
        static const size_t elem[9] = {4, 1, 4, 4, 4, 4, 4, 4, 4};
        return elem[c] * (size_t)L * (c == 0 ? (size_t)A : MA);
    }
    void place(Cols& c) {
        for (int b = 0; b < 9; ++b)
            if (lists[b]) o_list[b] = c.put(lists[b], list_bytes(b));
    }
    // g.rows: g.f with the row lists uploaded at d, and per_level (g: a ProfileArgs or a ProfileMarginArgs)
    template <class Args>
    void set_rows(Args& g, const char* d) const {
        g.rows = g.f;
        const auto row = [&](int b) { return (const void*)(d + o_list[b]); };
        if (lists[0]) g.rows.acc_cost = (const float*)row(0);
        if (lists[1]) g.rows.perf_present = (const uint8_t*)row(1);
        if (lists[2]) g.rows.perf_alpha = (const float*)row(2);
        if (lists[3]) g.rows.perf_beta = (const float*)row(3);
        if (lists[4]) g.rows.perf_gamma = (const float*)row(4);
        if (lists[5]) g.rows.perf_delta = (const float*)row(5);
        if (lists[6]) g.rows.perf_acc_count = (const int32_t*)row(6);
        if (lists[7]) g.rows.perf_max_batch = (const int32_t*)row(7);
        if (lists[8]) g.rows.perf_at_tokens = (const int32_t*)row(8);
        g.per_level = per_level;
    }
};


// The profile calls' keys with a perf column (DESIGN.md §3.15) of the rows rpm / in / out [L*S] into tk: per server
// the rows at which s is a load, grouped by (in, out) as in the workload calls; per group and accelerator a the rows
// at which (m, a) is present, grouped by the row's sizing key, one key row per key pair, whose accelerator and
// key-model go to key_acc and key_model.  skip(s, a) holds for a pair that keepAccelerator masks at every row.
template <class Skip>
void profile_keys(const HostFleet& hf, const ProfileRanks& pr, int L, const float* rpm, const int32_t* in,
                  const int32_t* out, Skip&& skip, TokenKeys& tk, std::vector<int>& key_acc,
                  std::vector<int>& key_model) {
    const int S = hf.S, A = hf.A, M = hf.M;
    LoadUses uses;                                              // (tokens key, row)
    std::vector<std::pair<std::array<uint64_t, 3>, int>> prof;  // (sizing key, row)
    for (int s = 0; s < S; ++s) {
        const int m = hf.srv_model[s];
        if (m < 0 || m >= M || !hf.srv_has_target[s]) continue;
        load_groups(L, S, s, rpm, in, out, uses, [&](int ki, int ko, size_t u0, size_t u1) {
            for (int a = 0; a < A; ++a) {
                if (skip(s, a)) continue;
                const size_t k = (size_t)m * A + a;
                prof.clear();
                for (size_t u = u0; u < u1; ++u) {
                    const int t = uses[u].second, j = pr.rank_at(t, k);
                    if (j >= 0) prof.emplace_back(pr.sizing_key(k, j, hf.srv_max_batch[s], ko), t);
                }
                std::sort(prof.begin(), prof.end());
                for (size_t v = 0; v < prof.size(); ++v) {
                    if (v == 0 || prof[v].first != prof[v - 1].first) {
                        tk.add(s, ki, ko);
                        key_acc.push_back(a);
                        key_model.push_back(pr.moff[m] + pr.rank_at(prof[v].second, k));
                    }
                    tk.add_level(prof[v].second);
                }
            }
        });
    }
}
// Their key fleet: key row k is server tk.srv[k] at the key's tokens on key-model key_model[k], with
// keepAccelerator and current accelerator key_acc[k], so that phase 1 sizes that pair alone.
KeyFleet profile_key_fleet(const HostFleet& hf, const ProfileRanks& pr, const TokenKeys& tk,
                           const std::vector<int>& key_acc, const std::vector<int>& key_model) {
    KeyFleet kf(hf, tk.srv, tk.in, tk.out);
    HostFleet& kh = kf.hf;
    kf.own_ma = true;
    for (size_t k = 0; k < tk.srv.size(); ++k) {
        kh.srv_model[k] = key_model[k];
        kh.srv_keep_acc[k] = 1;
        kh.srv_cur_acc[k] = key_acc[k];
    }
    pr.fill(kh);
    return kf;
}

// ---- walks: the load intervals and the load margins -----------------------------------------------------------
// The servers whose accelerator no tick of a trace can change (DESIGN.md §3.13), as flags [S]: with keepAccelerator
// and a current accelerator other than "" only that accelerator is a candidate, and its load and zero-load
// candidates carry it unless min_replicas is 0 (a zero-load candidate is then ""); an unknown one has no candidate at
// all.  A nil winner keeps the current allocation, so neither ever moves.  A trace's records carry keepAccelerator on
// these servers only: trace_kernel applies the rest of the mask tick by tick.
std::vector<uint8_t> trace_pinned(const HostFleet& hf) {
    std::vector<uint8_t> pin(hf.S);
    for (int s = 0; s < hf.S; ++s) {
        const int cur = hf.srv_cur_acc[s];
        pin[s] = hf.srv_keep_acc[s] && cur != WVA_ACC_NONE && (cur == WVA_ACC_UNKNOWN || hf.srv_min_replicas[s] != 0);
    }
    return pin;
}

// Warps per block (up to 4) of a kernel that runs one warp per item with per_warp bytes of dynamic shared memory per
// warp, the block's bytes, and the kernel's opt-in to more than 48 KiB where it needs that.
template <class Kernel>
int warp_layout(wva_handle* h, Kernel kernel, size_t per_warp, const char* what, int& wpb, size_t& smem) {
    int optin = 0;
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
    if (per_warp > (size_t)optin) return h->fail(WVA_ERR_UNSUPPORTED, what);
    wpb = (int)std::max<size_t>(1, std::min<size_t>(4, (48u << 10) / std::max<size_t>(per_warp, 1)));
    smem = per_warp * wpb;
    if (smem > (48u << 10)) CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return WVA_OK;
}

// The first half of a walk call over n = L * S windows lo / hi [n] (rows of S), whose device lists the caller has
// begun to place in c: phase 1 over the servers with some window top > 0, on a trace honouring keepAccelerator on
// the pinned servers only (trace_pinned); the record block g.rec (rec_bytes) zeroed, so that a record the walk does
// not write reads back as zero bytes; and the rest of g, whose records and work list (item, cap) the caller has set.
// With kf (the workload margins), phase 1 runs on every row of that key fleet instead, whose keepAccelerator column
// the caller has set, and whose columns it has placed in c; g.cand_of_pair then has K * A entries.
int enqueue_walk_star(wva_handle* h, Cols& c, int L, const float* lo, const float* hi, bool trace, size_t rec_bytes,
                      WalkArgs& g, LoadStar& ls, const KeyFleet* kf = nullptr) {
    const HostFleet& hf = kf ? kf->hf : h->hf;
    const int S = hf.S, A = hf.A, n = h->hf.S * L;
    std::vector<char> loaded(S, kf != nullptr);
    if (!kf)
        for (int i = 0; i < n; ++i) loaded[i % S] |= hi[i] > 0.0f;
    const std::vector<uint8_t> pin = trace && !kf ? trace_pinned(hf) : std::vector<uint8_t>();
    std::vector<int> pairs;
    const size_t o_lo = c.put(lo, 4 * (size_t)n), o_hi = c.put(hi, 4 * (size_t)n), o_cop = c.take(4 * (size_t)S * A);
    int rc = prepare_load_star(
        h, hf, loaded, pairs, c,
        [&](char* p) {
            int* cop = (int*)(p + o_cop);
            std::fill(cop, cop + (size_t)S * A, -1);
            for (size_t j = 0; j < pairs.size(); ++j) cop[pairs[j]] = (int)j;
        },
        pin.empty() ? nullptr : pin.data());
    if (rc) return rc;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    if (g.items.cap > 0) CK(cudaMemsetAsync(h->d_cand_block.p, 0, rec_bytes, h->stream));
    const char* dl = (const char*)h->lg_tabs.lists.p;
    rc = enqueue_load_star(h, hf, kf ? kf->view(h->df, dl) : h->df, g.items.cap, ls);
    if (rc) return rc;
    g.ld = load_args(h, ls);
    g.cand_of_pair = (const int*)(dl + o_cop);
    g.lo = (const float*)(dl + o_lo);
    g.hi = (const float*)(dl + o_hi);
    g.items.count = (int*)h->d_ctrl.p + CTRL_COUNTER;
    g.status = (int*)h->d_ctrl.p + CTRL_FB_STATUS;
    return WVA_OK;
}

// The walk kernel over `warps` items, one warp each with per_warp bytes of dynamic shared memory (refused with
// `what` where that does not fit a block), its tail over g's work list, ev_k1 (the call's kernel time: phase 1, a
// trace's chain and the walk kernels) and the re-run of the tail's bails (fallback over fb).
template <class Args>
int launch_walk(wva_handle* h, void (*walk)(Args), void (*tail)(Args), void (*fallback)(Args, FbRun), const Args& g,
                int warps, size_t per_warp, const char* what, const FbRun& fb) {
    int wpb = 0;
    size_t smem = 0;
    const int rc = warp_layout(h, walk, per_warp, what, wpb, smem);
    if (rc) return rc;
    walk<<<(unsigned)((warps + wpb - 1) / wpb), 32 * wpb, smem, h->stream>>>(g);
    const long long tail_blocks = std::min<long long>((long long)h->sm_count * 8, ((long long)g.items.cap + 255) / 256);
    tail<<<(unsigned)tail_blocks, 256, 0, h->stream>>>(g);
    h->launches += 2;
    CK(cudaEventRecord(h->ev_k1, h->stream));
    launch_fallback(h, fallback, g, fb);
    CK(cudaGetLastError());
    return WVA_OK;
}

// The end of a walk call from the upload on.  The call's device columns `cols` and then the work list [n_rec] live
// in h->d_iv, and the columns taken with a host destination come back to it; the n_rec records form one candidate
// block, copied back with `copy`.  enqueue(w, d, rec_bytes) runs under run_host, with d = h->d_iv.p and w the walk
// arguments' records and work list.  The block then goes back as recs.size() lists of equal length, one per entry.
template <class Enqueue>
int run_walk(wva_handle* h, const wva_fleet* fleet, Cols& cols, size_t n_rec, bool copy,
             std::initializer_list<const wva_allocs*> recs, Enqueue&& enqueue) {
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    const size_t o_items = cols.take(8 * n_rec);
    CK(h->d_iv.ensure(cols.bytes));
    char* d = (char*)h->d_iv.p;
    HostCall c{n_rec, copy, false, &cols, d};
    rc = run_host(h, c, [&](const AllocCols& dc, const AllocCols&) {
        WalkArgs w{};
        w.rec = dc;
        w.items = FbList{nullptr, (unsigned long long*)(d + o_items), (int)n_rec};
        return enqueue(w, d, c.bc.bytes);
    });
    // no single solution to summarise (upload_fleet cleared last_kind)
    if (rc) return rc;
    size_t k = 0;
    if (copy)
        for (const wva_allocs* r : recs) scatter_block(c.cand_host, sub_block(c.bc, k++, n_rec / recs.size()), r);
    return WVA_OK;
}

// ---- load intervals: where each server's load-grid winner changes in [lo, hi] ---------------------------------
// Phase 1 over the servers with hi > 0, interval_kernel, interval_tail and interval_fallback.  lo / hi [S] are the
// caller's bounds; g holds the call's device output columns, records and work list.
int enqueue_load_intervals(wva_handle* h, const float* lo, const float* hi, IntervalArgs& g, size_t rec_bytes) {
    const int S = h->hf.S;
    Cols c(16);
    LoadStar ls;
    int rc = enqueue_walk_star(h, c, 1, lo, hi, false, rec_bytes, g, ls);
    if (rc) return rc;
    // starts past a server's count read back as zero
    CK(cudaMemsetAsync(g.start, 0, 4 * (size_t)S * g.M, h->stream));
    if (S == 0) return WVA_OK;
    // one warp per server, A accelerator states per warp in shared memory
    return launch_walk(h, interval_kernel, interval_tail, interval_fallback, g, S, sizeof(IvAcc) * (size_t)h->hf.A,
                       "too many accelerators for the interval kernel's shared memory", ls.fb2);
}

// ---- load margins: the stretch around each level's rate on which the load-grid winner keeps its decision -------
static_assert(MG_LO_OPEN == WVA_MARGIN_LO_OPEN && MG_HI_OPEN == WVA_MARGIN_HI_OPEN &&
              MG_TRUNCATED == WVA_MARGIN_TRUNCATED, "margin flags");

// margin_kernel, margin_tail and margin_fallback of g (the Trace instantiations on a trace, after margin_chain): one
// warp per (level, server), A accelerator states and stretch starts per warp in shared memory.  Args is MarginArgs,
// or TokenMarginArgs, ProfileMarginArgs or SloMarginArgs for the workload, profile and SLO margins.
template <class Args>
int launch_margins(wva_handle* h, const Args& g, bool trace, const FbRun& fb) {
    const size_t per_warp = (sizeof(IvAcc) + sizeof(float)) * (size_t)h->hf.A;
    const char* what = "too many accelerators for the margin kernel's shared memory";
    if (!trace)
        return launch_walk(h, margin_kernel<false>, margin_tail<false>, margin_fallback<false>, g, g.n, per_warp, what,
                           fb);
    // one warp per server, A accelerator states per warp in shared memory
    void (*chain)(Args) = margin_chain;
    int wpb = 0;
    size_t smem = 0;
    const int rc = warp_layout(h, chain, sizeof(IvAcc) * (size_t)h->hf.A,
                               "too many accelerators for the margin chain's shared memory", wpb, smem);
    if (rc) return rc;
    chain<<<(unsigned)((h->hf.S + wpb - 1) / wpb), 32 * wpb, smem, h->stream>>>(g);
    h->launches++;
    return launch_walk(h, margin_kernel<true>, margin_tail<true>, margin_fallback<true>, g, g.n, per_warp, what, fb);
}

// Phase 1 over the servers with some window top > 0, then the margin kernels.  rate / lo / hi [L*S] are the caller's
// rows (rate NULL: the fleet's own column); g holds the call's device output columns, records and work list.
//
// With `trace` (wva_load_margin_trace, DESIGN.md §3.21) row t is tick t against c_t.  Phase 1 then honours
// keepAccelerator on the pinned servers only (trace_pinned): an unpinned server's chain can lift the mask at a later
// tick.  margin_chain writes c_t into g's c_t columns before the margin kernels read them through mg_view.
//
// With `tokens` (the workload margins, DESIGN.md §3.22) row l also has its own tokens, in / out [L*S] (NULL: the
// fleet's own column).  Size, lambda* and rateStar read the tokens but not the rate (§3.12), so phase 1 runs on the
// workload calls' key fleet: one row per distinct (server, in, out) over the rows whose window top is above 0 and
// whose tokens class a pair as a load (workload_keys with the window tops as its rates; on a trace with
// keepAccelerator on the pinned servers only).  The key column [L*S] names each row's key (-1: none), and the
// kernels read the rows' tokens through the row's view of the resident fleet.
//
// With `prof` (the profile margins, DESIGN.md §3.23) row l also has its own acc_cost and perf_* columns (ProfileRanks'
// layout; a NULL column is the fleet's own).  Price and AccCount enter only the cost, so without a perf column the
// keys are the workload margins' and the kernels price every record at its row.  With one, a load pair's record at
// row l is fixed by (s, a, in, out, the row's alpha .. delta and N), and the keys are the profile trace's
// (profile_keys, with the window tops as rates): one key row per key pair, so the key column [L*S*A] names each
// (row, server, accelerator)'s key row (-1: none).  keepAccelerator masks a pair at every row on the grid, and on a
// trace only on the pinned servers.
//
// With `slo` (the SLO margins, DESIGN.md §3.24) row l also has its own ITL, TTFT and TPS targets (NULL: the fleet's
// own column).  Size reads the ITL and TTFT targets and whether TPS is positive, and the tail's totalRate reads the
// TPS target, none of them the rate, so the keys are the workload margins' refined by the row's target bits
// (workload_keys with the target rows), and the key fleet carries each key's targets.  The kernels read the rows'
// targets through the row's view.
int enqueue_load_margins(wva_handle* h, int L, const float* rate, const int32_t* in, const int32_t* out, bool tokens,
                         const wva_profile_rows* prof, const TargetRows* slo, const float* lo, const float* hi,
                         ProfileMarginArgs& g, size_t rec_bytes, bool trace) {
    const HostFleet& hf = h->hf;
    const int S = hf.S, A = hf.A;
    Cols c(16);
    RowLists lists{hf, L, c};
    lists.put_rpm(rate);
    TokenKeys tk;
    std::optional<KeyFleet> kf;
    std::optional<ProfileRanks> pr;
    std::vector<int> key;
    size_t o_key = 0;
    if (tokens) {
        lists.put_tokens(in, out);
        if (slo) lists.put_targets(slo->itl, slo->ttft, slo->tps);
        const TargetRows tg{lists.itl.host, lists.ttft.host, lists.tps.host};
        const std::vector<uint8_t> pin = trace ? trace_pinned(hf) : std::vector<uint8_t>();
        if (prof) pr.emplace(hf, L, *prof);
        if (pr && pr->perf_rows) {
            std::vector<int> key_acc, key_model;
            profile_keys(hf, *pr, L, hi, lists.in.host, lists.out.host,
                         [&](int s, int a) {
                             const int cur = hf.srv_cur_acc[s];
                             return (trace ? pin[s] : hf.srv_keep_acc[s] && cur != WVA_ACC_NONE) && cur != a;
                         },
                         tk, key_acc, key_model);
            // the keys' pairs are indexed in int32 on the device
            if ((long long)tk.srv.size() * A >= (1ll << 31))
                return h->fail(WVA_ERR_UNSUPPORTED, "profile margins: too many key pairs for one call (K*A >= 2^31)");
            kf.emplace(profile_key_fleet(hf, *pr, tk, key_acc, key_model));
            key.assign((size_t)L * S * A, -1);
            for (size_t k = 0; k < tk.srv.size(); ++k)
                for (int j = tk.lev_off[k]; j < tk.lev_off[k + 1]; ++j)
                    key[((size_t)tk.lev[j] * S + tk.srv[k]) * A + key_acc[k]] = (int)k;
        } else {
            kf.emplace(workload_keys(hf, L, hi, lists.in.host, lists.out.host, trace ? pin.data() : nullptr, tk,
                                     slo ? &tg : nullptr));
            // the keys' pairs are indexed in int32 on the device
            if ((long long)tk.srv.size() * A >= (1ll << 31))
                return h->fail(WVA_ERR_UNSUPPORTED,
                               slo ? "SLO margins: too many keys for one call (K*A >= 2^31)"
                                   : "workload margins: too many token keys for one call (K*A >= 2^31)");
            key.assign((size_t)L * S, -1);
            for (size_t k = 0; k < tk.srv.size(); ++k)
                for (int j = tk.lev_off[k]; j < tk.lev_off[k + 1]; ++j) key[(size_t)tk.lev[j] * S + tk.srv[k]] = (int)k;
        }
        o_key = c.put(key.data(), 4 * key.size());
        kf->place(c);
        if (pr) pr->place(c);
    }
    LoadStar ls;
    int rc = enqueue_walk_star(h, c, L, lo, hi, trace, rec_bytes, g, ls, kf ? &*kf : nullptr);
    if (rc) return rc;
    if (g.n == 0) return WVA_OK;
    const char* d = (const char*)h->lg_tabs.lists.p;
    g.rate = lists.rpm.dev(d);
    if (!tokens) return launch_margins(h, static_cast<const MarginArgs&>(g), trace, ls.fb2);
    g.f = h->df;
    g.key = (const int*)(d + o_key);
    g.in_tokens = lists.in.dev(d);
    g.out_tokens = lists.out.dev(d);
    if (slo) {
        const SloMarginArgs sg{g, lists.itl.dev(d), lists.ttft.dev(d), lists.tps.dev(d)};
        return launch_margins(h, sg, trace, ls.fb2);
    }
    if (!pr) return launch_margins(h, static_cast<const TokenMarginArgs&>(g), trace, ls.fb2);
    pr->set_rows(g, d);
    g.pair_key = pr->perf_rows ? g.key : nullptr;
    return launch_margins(h, g, trace, ls.fb2);
}

// wva_load_margins, or with `trace` wva_load_margin_trace; with `tokens` wva_workload_margins or
// wva_workload_margin_trace (in / out: NULL is the fleet's own column), and with `prof` as well
// wva_profile_margins or wva_profile_margin_trace, or with `slo` (its lists NULL: the fleet's own column)
// wva_slo_margins or wva_slo_margin_trace.  All but wva_load_margins require the rate rows.
int load_margins_call(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                      const int32_t* in_tokens, const int32_t* out_tokens, bool tokens, const wva_profile_rows* prof,
                      const TargetRows* slo, const float* rpm_lo, const float* rpm_hi, wva_margins* out, bool trace) {
    if (!h) return WVA_ERR_BAD_ARG;
    if (!out) return h->fail(WVA_ERR_BAD_ARG, "out is NULL");
    if (n_levels < 0) return h->fail(WVA_ERR_BAD_ARG, trace ? "negative tick count" : "negative level count");
    if (const char* what = fleet_problem(fleet)) return h->fail(WVA_ERR_BAD_ARG, what);
    const int S = fleet->n_servers, L = n_levels;
    // three records per (level, server), each indexed in int32
    if (3ll * S * L >= (1ll << 31))
        return h->fail(WVA_ERR_UNSUPPORTED, "load margins too large for one call (>= 2^31 records)");
    if (prof && (long long)L * fleet->n_models * fleet->n_acc >= (1ll << 31))
        return h->fail(WVA_ERR_UNSUPPORTED, "profile margins too large for one call (>= 2^31 row entries)");
    const int n = S * L;
    if (n > 0 && (!rpm_lo || !rpm_hi || !out->lo_rpm || !out->hi_rpm || !out->flags))
        return h->fail(WVA_ERR_BAD_ARG, "NULL window or output column");
    if (n > 0 && (trace || tokens) && !arrival_rpm) return h->fail(WVA_ERR_BAD_ARG, "NULL arrival rate rows");
    for (int i = 0; i < n; ++i) {
        const float r = arrival_rpm ? arrival_rpm[i] : fleet->srv_arrival_rpm[i % S], lo = rpm_lo[i], hi = rpm_hi[i];
        if (!std::isfinite(r) || !std::isfinite(lo) || !std::isfinite(hi) || r < 0.0f || lo < 0.0f || hi < 0.0f ||
            lo > r || r > hi)
            return h->fail(WVA_ERR_BAD_ARG, "rate or window NaN, infinite or negative, or the rate outside its window");
    }
    Cols cols(16);
    const size_t o_lo = cols.take(4 * (size_t)n, out->lo_rpm), o_hi = cols.take(4 * (size_t)n, out->hi_rpm),
                 o_flags = cols.take((size_t)n, out->flags);
    const size_t o_cur = trace ? cols.take(12 * (size_t)n) : 0;  // a trace's c_t: acc, replicas, cost [n] each
    return run_walk(h, fleet, cols, 3 * (size_t)n, n > 0, {&out->at, &out->below, &out->above},
                    [&](const WalkArgs& w, char* d, size_t rec_bytes) {
                        ProfileMarginArgs g{TokenMarginArgs{MarginArgs{w}}};
                        g.n = n;
                        g.lo_out = (float*)(d + o_lo);
                        g.hi_out = (float*)(d + o_hi);
                        g.flags = (uint8_t*)(d + o_flags);
                        if (trace) {
                            g.cur_acc = (int*)(d + o_cur);
                            g.cur_replicas = (int*)(d + o_cur) + n;
                            g.cur_cost = (float*)(d + o_cur) + 2 * (size_t)n;
                        }
                        return enqueue_load_margins(h, L, arrival_rpm, in_tokens, out_tokens, tokens, prof, slo,
                                                    rpm_lo, rpm_hi, g, rec_bytes, trace);
                    });
}

// ---- SLO grid: CreateAllocation and the unlimited winner at every listed (ITL, TTFT, TPS) target row -----------
// A bisection reads only its own target (DESIGN.md §3.11), so phase 1 runs each distinct (server, search, target
// bits) key once per load pair of the server, in search mode; phase 2 (slo_kernel, slo_fallback) is the tail per
// (load pair, level).  A key exists where some level needs it: the level's three targets are not negative
// (TargetPerf.check makes the pair nil before any search), the target is > 0 (0, -0 and NaN disable a search) and
// the server has load pairs.  Lists, tables (lg_tabs, shared with the load grid and the load intervals) and the
// search records (d_slo) are rebuilt on every call.  itl / ttft / tps [L*S] are the caller's rows; cand ([L*S*A])
// and winners ([L*S]) are device columns.
//
// SloKeys holds phase 1's searches for the SLO grid and the SLO trace: a search is fixed by (key row, accelerator,
// which search, target bits), where a key row is one (server, tokens) with the rows at which it applies.  The grid's
// key rows are the resident servers, each at every level; the trace's are the workload trace's token keys, each at
// the ticks that use its tokens under load.  build() lists, per key row with load pairs, its distinct (search, target
// bits) in that order and crosses them with the row's load pairs (the tail's candidates `pairs`, descending N, one
// N-entry table each): the search candidates, still in descending N.  The key of each (row, server, search) and the
// search candidates travel in the call's upload image (place, write); enqueue() runs the searches in search mode over
// the tables of lg_tabs, records in d_slo.
struct SloKeys {
    std::vector<int> key;        // [2 * L * S] key of (row l, server s, search w) at (l * S + s) * 2 + w; -1: none
    std::vector<uint8_t> key_w;  // per key: its search (0: TTFT, 1: ITL) ...
    std::vector<float> key_t;    // ... and target
    std::vector<std::pair<int, int>> sc;  // the search candidates (key, pair)
    std::vector<int> tab_of;              // a pair's table index
    std::vector<long long> tab_entry;     // a table's first entry
    size_t o_key = 0, o_pair = 0, o_N = 0, o_rec = 0, o_idx = 0, o_off = 0, o_tgt = 0, o_which = 0;
    AllocCols srch{};  // the search records by key * A + a, set by enqueue

    // R key rows: row r is server srv(r) and applies at the rows ticks(r, fn) hands to fn, ascending; pairs r * A + a.
    // Refuses 2^31 or more search records (`what` names the call).
    template <class Srv, class Ticks>
    int build(wva_handle* h, const char* what, int L, int S, int A, int R, Srv&& srv, Ticks&& ticks,
              const float* itl, const float* ttft, const float* tps, const std::vector<int>& pairs,
              const std::vector<int>& Ns) {
        tab_of.assign((size_t)R * A, -1);
        tab_entry.resize(pairs.size());
        long long entries = 0;
        for (size_t t = 0; t < pairs.size(); ++t) {
            tab_of[pairs[t]] = (int)t;
            tab_entry[t] = entries;
            entries += Ns[t];
        }
        std::vector<int> n_load(R, 0);
        for (int p : pairs) n_load[p / A]++;
        // a row's keys are key_begin[r] .. key_begin[r + 1] - 1
        std::vector<int> key_begin(R + 1, 0);
        key.assign(2 * (size_t)L * S, -1);
        std::vector<std::pair<uint64_t, size_t>> uses;  // (search << 32 | target bits, index into key)
        for (int r = 0; r < R; ++r) {
            key_begin[r] = (int)key_w.size();
            if (!n_load[r]) continue;
            const int s = srv(r);
            uses.clear();
            ticks(r, [&](int l) {
                const size_t i = (size_t)l * S + s;
                if (itl[i] < 0.0f || ttft[i] < 0.0f || tps[i] < 0.0f) return;
                for (int w = 0; w < 2; ++w) {
                    const float t = w == 0 ? ttft[i] : itl[i];
                    if (!(t > 0.0f)) continue;
                    uint32_t bits;
                    memcpy(&bits, &t, 4);
                    uses.emplace_back((uint64_t)w << 32 | bits, 2 * i + w);
                }
            });
            std::sort(uses.begin(), uses.end());
            for (size_t u = 0; u < uses.size(); ++u) {
                if (u == 0 || uses[u].first != uses[u - 1].first) {
                    const uint32_t bits = (uint32_t)uses[u].first;
                    float t;
                    memcpy(&t, &bits, 4);
                    key_w.push_back((uint8_t)(uses[u].first >> 32));
                    key_t.push_back(t);
                }
                key[uses[u].second] = (int)key_w.size() - 1;
            }
            // at most 2 * L * S keys in all; the search candidates are fewer than the records
            if ((long long)key_w.size() * A >= (1ll << 31)) {
                const std::string msg = std::string(what) + " with 2^31 or more search records in one call";
                return h->fail(WVA_ERR_UNSUPPORTED, msg.c_str());
            }
        }
        key_begin[R] = (int)key_w.size();
        // the load pairs in their order (descending N), each with its row's keys
        for (int p : pairs)
            for (int k = key_begin[p / A]; k < key_begin[p / A + 1]; ++k) sc.emplace_back(k, p);
        return WVA_OK;
    }
    void place(Cols& c) {
        const size_t n = sc.size();
        o_key = c.put(key.data(), 4 * key.size());
        o_pair = c.take(4 * n);
        o_N = c.take(4 * n);
        o_rec = c.take(4 * n);
        o_idx = c.take(4 * n);
        o_off = c.take(8 * n);
        o_tgt = c.take(4 * n);
        o_which = c.take(n);
    }
    void write(char* p, const std::vector<int>& Ns, int A) const {
        for (size_t j = 0; j < sc.size(); ++j) {
            const int k = sc[j].first, pair = sc[j].second, a = pair % A, t = tab_of[pair];
            ((int*)(p + o_pair))[j] = pair;
            ((int*)(p + o_N))[j] = Ns[t];
            ((int*)(p + o_rec))[j] = k * A + a;
            ((int*)(p + o_idx))[j] = t;
            ((long long*)(p + o_off))[j] = tab_entry[t];
            ((float*)(p + o_tgt))[j] = key_t[k];
            ((uint8_t*)(p + o_which))[j] = key_w[k];
        }
    }
    // d_slo for the records; call before enqueue
    int reserve(wva_handle* h) {
        const size_t n_srec = key_w.size() * (size_t)h->hf.A;
        CK(h->d_slo.ensure(5 * n_srec + 16));
        srch = AllocCols{};
        srch.max_rate = (float*)h->d_slo.p;
        srch.feasible = (uint8_t*)h->d_slo.p + 4 * n_srec;
        return WVA_OK;
    }
    // phase 1: the searches on fleet f (whose tables are lg_tabs', uploaded at d)
    int enqueue(wva_handle* h, const DevFleet& f, const char* d) const {
        const PairTables& pt = h->lg_tabs;
        SizeArgs g = size_args(f, pt, srch);
        g.cand_pair = (const int*)(d + o_pair);
        g.cand_N = (const int*)(d + o_N);
        g.n_cand = (int)sc.size();
        g.tab_off = (const long long*)(d + o_off);
        g.place = CandPlace{(const int*)(d + o_idx), (const int*)(d + o_rec)};
        return enqueue_candidates(h, g, pt.len_max, SIZE_SEARCH,
                                  SearchCols{(const uint8_t*)(d + o_which), (const float*)(d + o_tgt)});
    }
};

int enqueue_slo_grid(wva_handle* h, int L, const float* itl, const float* ttft, const float* tps,
                     const AllocCols& cand, const AllocCols& winners) {
    const HostFleet& hf = h->hf;
    const int S = hf.S, A = hf.A;
    // the tail's candidates: every load pair (none without levels), descending N, one N-entry table each
    std::vector<int> pairs, Ns;
    if (L > 0) {
        const int rc =
            sorted_pairs(h, hf, [&](int s, int a) { return hf.pair_class(s, a, true) == PAIR_LOAD; }, pairs, Ns);
        if (rc) return rc;
    }
    Cols c(16);
    RowLists lists{hf, L, c};
    lists.put_targets(itl, ttft, tps);
    // one key row per server, at every level
    SloKeys sk;
    int rc = sk.build(
        h, "SLO grid", L, S, A, S, [](int s) { return s; },
        [&](int, auto&& fn) {
            for (int l = 0; l < L; ++l) fn(l);
        },
        itl, ttft, tps, pairs, Ns);
    if (rc) return rc;
    sk.place(c);
    rc = upload_tables(h, h->lg_tabs, pairs, Ns, true, c, [&](char* p) { sk.write(p, Ns, A); });
    if (rc) return rc;
    const PairTables& pt = h->lg_tabs;
    const char* d = (const char*)pt.lists.p;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    const long long n_items = (long long)pt.n * L;
    FbRun fb2;
    rc = prepare_tail(h, h->df, n_items, fb2);
    if (rc) return rc;
    rc = sk.reserve(h);
    if (rc) return rc;
    launch_records(h, (long long)S * A * L, trivial_kernel, h->df, cand, lists.load(d), L);
    // phase 1: the searches
    rc = sk.enqueue(h, h->df, d);
    if (rc) return rc;
    // phase 2: the tail per (load pair, level)
    if (n_items > 0) {
        SloArgs la{};
        set_tables(la, h->df, pt);
        la.slo_itl = lists.itl.dev(d);
        la.slo_ttft = lists.ttft.dev(d);
        la.slo_tps = lists.tps.dev(d);
        la.key = (const int*)(d + sk.o_key);
        la.srch = sk.srch;
        la.L = L;
        la.counter = (unsigned*)h->d_ctrl.p + CTRL_COUNTER;
        la.status = (int*)h->d_ctrl.p + CTRL_FB_STATUS;
        la.cand = cand;
        la.fb = fb2.list;
        rc = launch_tail(h, slo_kernel, slo_fallback, la, (n_items + 31) / 32, fb2);
        if (rc) return rc;
    }
    enqueue_level_winners(h, cand, winners, L, false);
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- workload grid: CreateAllocation and the unlimited winner at every listed (rate, in, out) row --------------
// The workload grid's tail (workload_kernel, then workload_fallback) after phase 1 (ls): g's key and level lists and
// g.n_items items, at the rates level_rpm [L * g.S], into cand.  ev_k1 is recorded after workload_kernel: the
// call's kernel time covers both phases.
int enqueue_workload_tail(wva_handle* h, const LoadStar& ls, WorkloadArgs& g, const float* level_rpm, int L,
                          const AllocCols& cand) {
    if (g.n_items <= 0) return WVA_OK;
    g.ld = load_args(h, ls);
    g.ld.level_rpm = level_rpm;
    g.ld.L = L;
    g.ld.counter = (unsigned*)h->d_ctrl.p + CTRL_COUNTER;
    g.ld.cand = cand;
    return launch_tail(h, workload_kernel, workload_fallback, g, ((long long)g.n_items + 31) / 32, ls.fb2);
}

// QueueAnalyzer.Size, lambda* and rateStar read a server's tokens but not its rate (DESIGN.md §3.12), so phase 1
// is the load grid's, run once on the key fleet: one row per distinct (server, in_tokens, out_tokens) that some
// level uses under load (rate not negative and not 0, NaN and +Inf included; in_tokens >= 0; out_tokens >= 1).
// Phase 2 (workload_kernel, workload_fallback) is the load grid's tail per (key candidate, level of the key).  The
// lists, the key fleet's server columns and the tables go into lg_tabs, rebuilt on every call.  Then the unlimited
// winner of every level.  rpm / in / out [L*S] are the caller's rows (a NULL token list: the fleet's own column at
// every row); cand ([L*S*A]) and winners ([L*S]) are device columns.
//
// With `trace` (the workload trace, DESIGN.md §3.13) the records carry keepAccelerator on the pinned servers only
// (trace_pinned), in trivial_kernel and in the key fleet alike.  trace_kernel's chain then picks the winners: one
// thread per server applies the mask against its current allocation, picks the winner and advances.
int enqueue_workload(wva_handle* h, int L, const float* rpm, const int32_t* in, const int32_t* out,
                     const AllocCols& cand, const AllocCols& winners, bool trace) {
    const HostFleet& hf = h->hf;
    const int S = hf.S, A = hf.A;
    Cols c(16);
    RowLists lists{hf, L, c};
    lists.put_rpm(rpm);
    lists.put_tokens(in, out);
    const std::vector<uint8_t> pin = trace ? trace_pinned(hf) : std::vector<uint8_t>();
    const size_t o_pin = trace ? c.put(pin.data(), S) : 0;
    // the keys: at most L * S, so fewer than 2^31 key candidates
    TokenKeys tk;
    KeyFleet kf = workload_keys(hf, L, rpm, lists.in.host, lists.out.host, trace ? pin.data() : nullptr, tk);
    const int K = (int)tk.srv.size();
    kf.place(c);
    tk.place(c, (size_t)K * A);
    std::vector<int> pairs;
    int rc = prepare_load_star(h, kf.hf, std::vector<char>(K, 1), pairs, c, [&](char* p) { tk.write(p, pairs, A); });
    if (rc) return rc;
    const char* d = (const char*)h->lg_tabs.lists.p;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    DevFleet tf = h->df;
    if (trace) tf.srv_keep_acc = (const uint8_t*)(d + o_pin);
    launch_records(h, (long long)S * A * L, trivial_kernel, tf, cand, lists.load(d), L);
    LoadStar ls;
    rc = enqueue_load_star(h, kf.hf, kf.view(h->df, d), tk.n_items, ls);
    if (rc) return rc;
    WorkloadArgs g = tk.args(d, S);
    rc = enqueue_workload_tail(h, ls, g, lists.rpm.dev(d), L, cand);
    if (rc) return rc;
    enqueue_level_winners(h, cand, winners, L, trace);
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- SLO trace: the reconcile replayed over ticks of load and service-class targets (DESIGN.md §3.17) -------------
// Size, lambda* and rateStar read the tokens but not the rate (§3.12), and each bisection reads only its own target
// (§3.11), so a search is fixed by (server, accelerator, in, out, which search, target bits).  The key rows are the
// workload trace's (server, in, out) rows under load, on a key fleet that keeps keepAccelerator only on the pinned
// servers; SloKeys runs each distinct search of a key row once per load pair of the row.  The tail (slo_trace_kernel,
// slo_trace_fallback) then runs per (key candidate, tick of its row) at f_t, the workload trace's trivial_kernel writes
// the nil and zero-load records, and trace_kernel runs the chain.  The six row lists (NULL: the fleet's own column at
// every tick) are in the call's upload image; lists, key fleet columns and tables go into lg_tabs, rebuilt on every
// call.  cand ([L*S*A]) and winners ([L*S]) are device columns.
int enqueue_slo_trace(wva_handle* h, int L, const float* rpm, const int32_t* in, const int32_t* out, const float* itl,
                      const float* ttft, const float* tps, const AllocCols& cand, const AllocCols& winners) {
    const HostFleet& hf = h->hf;
    const int S = hf.S, A = hf.A;
    Cols c(16);
    RowLists lists{hf, L, c};
    lists.put_rpm(rpm);
    lists.put_tokens(in, out);
    lists.put_targets(itl, ttft, tps);
    const std::vector<uint8_t> pin = trace_pinned(hf);
    const size_t o_pin = c.put(pin.data(), S);
    // the key rows: at most L * S
    TokenKeys tk;
    KeyFleet kf = workload_keys(hf, L, lists.rpm.host, lists.in.host, lists.out.host, pin.data(), tk);
    const int K = (int)tk.srv.size();
    // the tail's candidates: the key fleet's load pairs, descending N, one N-entry table each
    const HostFleet& kh = kf.hf;
    std::vector<int> pairs, Ns;
    int rc = sorted_pairs(h, kh, [&](int k, int a) { return kh.pair_class(k, a, true) == PAIR_LOAD; }, pairs, Ns);
    if (rc) return rc;
    SloKeys sk;
    rc = sk.build(
        h, "SLO trace", L, S, A, K, [&](int k) { return tk.srv[k]; },
        [&](int k, auto&& fn) {
            for (int j = tk.lev_off[k]; j < tk.lev_off[k + 1]; ++j) fn(tk.lev[j]);
        },
        lists.itl.host, lists.ttft.host, lists.tps.host, pairs, Ns);
    if (rc) return rc;
    kf.place(c);
    tk.place(c, pairs.size());
    sk.place(c);
    rc = upload_tables(h, h->lg_tabs, pairs, Ns, true, c, [&](char* p) {
        tk.write(p, pairs, A);
        sk.write(p, Ns, A);
    });
    if (rc) return rc;
    const PairTables& pt = h->lg_tabs;
    const char* d = (const char*)pt.lists.p;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    const DevFleet kd = kf.view(h->df, d);
    FbRun fb2;
    rc = prepare_tail(h, kd, tk.n_items, fb2);
    if (rc) return rc;
    rc = sk.reserve(h);
    if (rc) return rc;
    // the workload trace's nil and zero-load records: keepAccelerator on the pinned servers only, no target read
    DevFleet tf = h->df;
    tf.srv_keep_acc = (const uint8_t*)(d + o_pin);
    launch_records(h, (long long)S * A * L, trivial_kernel, tf, cand, lists.load(d), L);
    // phase 1: the searches
    rc = sk.enqueue(h, kd, d);
    if (rc) return rc;
    // phase 2: the tail per (key candidate, tick of its key row)
    if (tk.n_items > 0) {
        SloTraceArgs g{};
        g.w = tk.args(d, S);
        set_tables(g.w.ld, kd, pt);
        g.w.ld.level_rpm = lists.rpm.dev(d);
        g.w.ld.L = L;
        g.w.ld.counter = (unsigned*)h->d_ctrl.p + CTRL_COUNTER;
        g.w.ld.cand = cand;
        g.w.ld.fb = fb2.list;
        g.f = h->df;
        g.tick_in = lists.in.dev(d);
        g.tick_out = lists.out.dev(d);
        g.slo_itl = lists.itl.dev(d);
        g.slo_ttft = lists.ttft.dev(d);
        g.slo_tps = lists.tps.dev(d);
        g.key = (const int*)(d + sk.o_key);
        g.srch = sk.srch;
        g.status = (int*)h->d_ctrl.p + CTRL_FB_STATUS;
        rc = launch_tail(h, slo_trace_kernel, slo_trace_fallback, g, ((long long)tk.n_items + 31) / 32, fb2);
        if (rc) return rc;
    }
    enqueue_level_winners(h, cand, winners, L, true);
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- profile grid: CreateAllocation and the unlimited winner at every listed (acc_cost, perf) row (DESIGN.md §3.14)
// CreateAllocation reads the accelerator's cost and AccCount only in the allocation's cost, so a load pair's record
// at level l is fixed by the pair and the row's (alpha, beta, gamma, delta, N).  The host ranks the distinct rows of
// each (m, a) that the levels use (present ones only: elsewhere no pair of m is a load), and builds a key fleet:
// key-model (m, j) holds the j-th distinct row of (m, a) at every accelerator a that has one, so its tables stay
// within L * M * A entries, and key row k is server key_srv[k] on one key-model, at the server's own load.  Per load
// pair (s, a) the rows with equal (alpha .. delta, N) share the lowest j's key.  Phase 1 and the workload grid's tail
// run on the key fleet with one "level" (its own rates), writing one record per key pair; profile_kernel then writes
// every level's records and the existing L-block unlimited_kernel the winners.  The lists, the row lists and the key
// fleet's columns go into lg_tabs, rebuilt on every call.  cand ([L*S*A]) and winners ([L*S]) are device columns.
int enqueue_profile_grid(wva_handle* h, int L, const wva_profile_rows& rows, const AllocCols& cand,
                         const AllocCols& winners) {
    const HostFleet& hf = h->hf;
    const int S = hf.S, A = hf.A;
    ProfileRanks pr(hf, L, rows);
    // Per load pair (s, a): one key_of entry per distinct row j of (m, a), pointing at the key record of the lowest
    // row with the same (alpha .. delta, N).  The key rows are (server, key-model) pairs numbered in server order;
    // need[k * A + a] marks the key pairs phase 1 sizes.
    std::vector<int> pair_off((size_t)S * A + 1, 0), key_of, key_srv, key_model;
    std::vector<char> need;
    std::vector<std::pair<std::array<uint64_t, 3>, int>> groups;  // ((alpha, beta), (gamma, delta), N), j
    std::vector<int> srv_js;
    for (int s = 0; s < S; ++s) {
        const int m = hf.srv_model[s];
        srv_js.clear();
        for (int a = 0; a < A; ++a) {
            const size_t pair = (size_t)s * A + a;
            pair_off[pair] = (int)key_of.size();
            // the pair's class at a level where it is present (elsewhere it is nil)
            if (hf.pair_class(s, a, true, hf.srv_arrival_rpm[s], true) != PAIR_LOAD) continue;
            const size_t k = (size_t)m * A + a;
            const int J = pr.row_off[k + 1] - pr.row_off[k], e0 = (int)key_of.size();
            groups.clear();
            for (int j = 0; j < J; ++j)
                groups.push_back({pr.sizing_key(k, j, hf.srv_max_batch[s], hf.srv_out_tokens[s]), j});
            std::sort(groups.begin(), groups.end());
            key_of.resize(key_of.size() + J);  // the representative row for now
            for (size_t u = 0; u < groups.size(); ++u) {
                const bool dup = u > 0 && groups[u].first == groups[u - 1].first;
                const int rep = dup ? key_of[e0 + groups[u - 1].second] : groups[u].second;
                key_of[e0 + groups[u].second] = rep;
                if (!dup) srv_js.push_back(rep);
            }
        }
        std::sort(srv_js.begin(), srv_js.end());
        srv_js.erase(std::unique(srv_js.begin(), srv_js.end()), srv_js.end());
        const int base = (int)key_srv.size();
        for (int j : srv_js) {
            key_srv.push_back(s);
            key_model.push_back(pr.moff[m] + j);
        }
        need.resize(key_srv.size() * A, 0);
        for (int a = 0; a < A; ++a) {
            const size_t pair = (size_t)s * A + a;
            const size_t end = a + 1 < A ? (size_t)pair_off[pair + 1] : key_of.size();
            for (size_t e = pair_off[pair]; e < end; ++e) {
                const int kr = base + (int)(std::lower_bound(srv_js.begin(), srv_js.end(), key_of[e]) - srv_js.begin());
                key_of[e] = kr * A + a;
                need[(size_t)kr * A + a] = 1;
            }
        }
    }
    pair_off[(size_t)S * A] = (int)key_of.size();
    const int K = (int)key_srv.size();  // at most L * S * A key pairs in all (checked by the caller)

    // the key fleet: key row k is server key_srv[k] on key-model key_model[k], at the server's own load
    std::vector<int> key_in(K), key_out(K);
    for (int k = 0; k < K; ++k) {
        key_in[k] = hf.srv_in_tokens[key_srv[k]];
        key_out[k] = hf.srv_out_tokens[key_srv[k]];
    }
    KeyFleet kf(hf, key_srv, key_in, key_out);
    HostFleet& kh = kf.hf;
    kf.own_ma = true;
    for (int k = 0; k < K; ++k) {
        kh.srv_arrival_rpm[k] = hf.srv_arrival_rpm[key_srv[k]];
        kh.srv_model[k] = key_model[k];
    }
    pr.fill(kh);
    std::vector<int> pairs, Ns;
    int rc = sorted_pairs(h, kh, [&](int k, int a) { return need[(size_t)k * A + a] != 0; }, pairs, Ns);
    if (rc) return rc;
    const int n = (int)pairs.size();

    // the key records: one per key pair, written by the workload grid's tail
    const Block kb = block_layout((size_t)K * A);
    CK(h->d_prof.ensure(kb.bytes + 16));
    const AllocCols key = block_cols(h->d_prof.p, kb);

    Cols c(16);
    kf.place(c);
    pr.place(c);
    const std::vector<int>& rank = pr.rank;
    const size_t o_rank = c.put(rank.data(), 4 * rank.size()), o_poff = c.put(pair_off.data(), 4 * pair_off.size()),
                 o_keyof = c.put(key_of.data(), 4 * key_of.size()), o_ksrv = c.take(4 * (size_t)K),
                 o_loff = c.take(4 * ((size_t)K + 1)), o_lev = c.take(4 * (size_t)K),
                 o_item = c.take(4 * ((size_t)n + 1));
    rc = upload_tables(h, h->lg_tabs, pairs, Ns, true, c, [&](char* p) {
        // the tail's one level: key k is server k of the key fleet, candidate e item e (written in place: building
        // them as TokenKeys costs the host measurably more at 10^5 keys)
        int* ksrv = (int*)(p + o_ksrv);
        int* loff = (int*)(p + o_loff);
        int* item = (int*)(p + o_item);
        std::iota(ksrv, ksrv + K, 0);
        std::iota(loff, loff + K + 1, 0);
        memset(p + o_lev, 0, 4 * (size_t)K);
        std::iota(item, item + n + 1, 0);
    });
    if (rc) return rc;
    const char* d = (const char*)h->lg_tabs.lists.p;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    const DevFleet kd = kf.view(h->df, d);
    LoadStar ls;
    rc = enqueue_load_star(h, kh, kd, n, ls);
    if (rc) return rc;
    WorkloadArgs t{};
    t.key_srv = (const int*)(d + o_ksrv);
    t.lev_off = (const int*)(d + o_loff);
    t.lev = (const int*)(d + o_lev);
    t.item_off = (const int*)(d + o_item);
    t.S = K;
    t.n_items = n;
    rc = enqueue_workload_tail(h, ls, t, kd.srv_arrival_rpm, 1, key);
    if (rc) return rc;
    ProfileArgs g{};
    g.f = h->df;
    pr.set_rows(g, d);
    g.rank = pr.perf_rows ? (const int*)(d + o_rank) : nullptr;
    g.pair_off = (const int*)(d + o_poff);
    g.key_of = (const int*)(d + o_keyof);
    g.key = key;
    g.cand = cand;
    g.L = L;
    launch_records(h, (long long)S * A * L, profile_kernel, g);
    enqueue_level_winners(h, cand, winners, L, false);
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- profile trace: the reconcile replayed over ticks of load and of (acc_cost, perf) rows (DESIGN.md §3.15) ------
// CreateAllocation reads neither the current allocation (§3.13) nor, outside the cost, the price and AccCount
// (§3.14).  So a load pair's record at tick t is fixed by its key (s, a, in_t, out_t, bits of alpha .. delta at row
// t, N at row t), and every tick is sized in one pass.  The workload grid's tail gives every candidate of a key row
// the row's tick list, so:
// - with a perf column given, the key fleet has one row per key pair: server s at the key's tokens on the
//   key-model (ProfileRanks) of a row of the key, with keepAccelerator and current accelerator a, so that
//   prepare_load_star sizes that pair alone;
// - with none, every accelerator of (s, in, out) has the same rows at every tick, and the key fleet is the workload
//   trace's: rows (s, in, out) on the fleet's own models, keepAccelerator kept on the pinned servers only.  So the
//   call sizes the same pairs, in the same order, with the same phase-1 work.
// Phase 1 and the workload grid's tail run unchanged and write each loaded (t, s, a) record in place;
// profile_trace_kernel then writes the nil and zero-load records and prices the tail's at row t, and the workload
// trace's trace_kernel runs the chain.  rpm / in / out [L*S] are the caller's rows (NULL: the fleet's own column at
// every tick); cand ([L*S*A]) and winners ([L*S]) are device columns.
//
// Without `trace` (the grid mode of the profile price thresholds, DESIGN.md §3.25) every row is a level against the
// fleet's own current allocation.  keepAccelerator then masks a pair at every row, as on the profile margins' grid:
// the keys skip it (profile_keys) or carry the fleet's own keepAccelerator (workload_keys without pins),
// profile_trace_kernel classes the records with the resident keepAccelerator, and unlimited_kernel picks each
// level's winners.  acc_count, when given, receives the device copy of the perf_acc_count row list (NULL without
// one), which stays in place until the next call.
int enqueue_profile_trace(wva_handle* h, int L, const float* rpm, const int32_t* in, const int32_t* out,
                          const wva_profile_rows& rows, const AllocCols& cand, const AllocCols& winners,
                          bool trace = true, const int32_t** acc_count = nullptr) {
    const HostFleet& hf = h->hf;
    const int S = hf.S, A = hf.A;
    Cols c(16);
    RowLists lists{hf, L, c};
    lists.put_rpm(rpm);
    lists.put_tokens(in, out);
    rpm = lists.rpm.host;  // from here on: the caller's lists or the tiled columns
    in = lists.in.host;
    out = lists.out.host;
    ProfileRanks pr(hf, L, rows);
    const std::vector<uint8_t> pin = trace ? trace_pinned(hf) : std::vector<uint8_t>();
    const size_t o_pin = trace ? c.put(pin.data(), S) : 0;
    // The keys.  Without a perf column: the workload trace's (s, in, out) rows (the workload grid's without
    // `trace`).  With one: profile_keys, a pinned server sizing its current pair alone.
    TokenKeys tk;
    std::vector<int> key_acc, key_model;  // with a perf column: key row k's accelerator and key-model
    if (pr.perf_rows) {
        profile_keys(hf, pr, L, rpm, in, out,
                     [&](int s, int a) {
                         const int cur = hf.srv_cur_acc[s];
                         return (trace ? pin[s] : hf.srv_keep_acc[s] && cur != WVA_ACC_NONE) && cur != a;
                     },
                     tk, key_acc, key_model);
        // at most L * S * A key rows; the key fleet's pair ids k * A + a are int
        if ((long long)tk.srv.size() * A >= (1ll << 31))
            return h->fail(WVA_ERR_UNSUPPORTED, trace
                               ? "profile trace too large for one call (>= 2^31 key pairs x accelerators)"
                               : "profile rows too large for one call (>= 2^31 key pairs x accelerators)");
    }
    KeyFleet kf = pr.perf_rows ? profile_key_fleet(hf, pr, tk, key_acc, key_model)
                               : workload_keys(hf, L, rpm, in, out, trace ? pin.data() : nullptr, tk);
    const int K = (int)tk.srv.size();
    HostFleet& kh = kf.hf;
    kf.place(c);
    pr.place(c);
    // the tail's candidates: one per key row with a perf column, up to A without
    tk.place(c, pr.perf_rows ? (size_t)K : (size_t)K * A);
    std::vector<int> pairs;
    int rc = prepare_load_star(h, kh, std::vector<char>(K, 1), pairs, c, [&](char* p) { tk.write(p, pairs, A); });
    if (rc) return rc;
    const char* d = (const char*)h->lg_tabs.lists.p;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    LoadStar ls;
    rc = enqueue_load_star(h, kh, kf.view(h->df, d), tk.n_items, ls);
    if (rc) return rc;
    WorkloadArgs g = tk.args(d, S);
    rc = enqueue_workload_tail(h, ls, g, lists.rpm.dev(d), L, cand);
    if (rc) return rc;
    ProfileTraceArgs r{};
    r.p.f = h->df;
    if (trace) r.p.f.srv_keep_acc = (const uint8_t*)(d + o_pin);
    pr.set_rows(r.p, d);
    r.p.cand = cand;
    r.p.L = L;
    r.rows = lists.load(d);
    launch_records(h, (long long)S * A * L, profile_trace_kernel, r);
    enqueue_level_winners(h, cand, winners, L, trace);
    if (acc_count) *acc_count = rows.perf_acc_count ? r.p.rows.perf_acc_count : nullptr;
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- price thresholds: the price of each accelerator at which each server's winner leaves it (DESIGN.md §3.16) --
// The inputs on which a pair's value can decrease as its price grows, so that its winning prices need not be one
// interval from 0: a penalty factor that is NaN, negative or infinite, or a non-finite current cost on a server
// that has a candidate (a pair wva_analyze does not class nil).  The first rule is the fleet's; the second is
// checked per row of L rows (the single call's one row is the fleet itself): at row l server s has the arrival rate
// rpm[l*S + s], the tokens in / out[l*S + s] (NULL: the fleet's own column), the models' perf_present
// present[(l*M + m)*A + a] (NULL: the fleet's own column) and the current allocation cur(l, s) -> (accelerator,
// cost).  Each returns its refusal, empty when there is none.
std::string price_factor_refusal(const HostFleet& hf) {
    const float f = hf.tun.accel_penalty_factor;
    return !(f >= 0.0f) || std::isinf(f) ? "penalty factor NaN, negative or infinite" : "";
}
template <class Cur>
std::string price_cost_refusal(const HostFleet& hf, int L, const float* rpm, const int32_t* in, const int32_t* out,
                               const uint8_t* present, const char* row, Cur&& cur) {
    const int S = hf.S;
    for (int l = 0; l < L; ++l)
        for (int s = 0; s < S; ++s) {
            const std::pair<int, float> c = cur(l, s);
            if (std::isfinite(c.second)) continue;
            const size_t i = (size_t)l * S + s;
            const int ki = in ? in[i] : hf.srv_in_tokens[s], ko = out ? out[i] : hf.srv_out_tokens[s];
            const int m = hf.srv_model[s];
            const bool known = m >= 0 && m < hf.M;
            for (int a = 0; a < hf.A; ++a)
                if (present ? hf.pair_class(s, a, true, rpm[i], ki, ko, c.first,
                                            known && present[((size_t)l * hf.M + m) * hf.A + a])
                            : hf.pair_class(s, a, true, rpm[i], ki, ko, c.first)) {
                    std::string what = "current cost NaN or infinite on a server with a candidate (server " +
                                       std::to_string(s);
                    return row ? what + ", " + row + " " + std::to_string(l) + ")" : what + ")";
                }
        }
    return "";
}
std::string price_refusal(const HostFleet& hf) {
    const std::string what = price_factor_refusal(hf);
    if (!what.empty()) return what;
    return price_cost_refusal(hf, 1, hf.srv_arrival_rpm.data(), nullptr, nullptr, nullptr, nullptr,
                              [&](int, int s) { return std::make_pair(hf.srv_cur_acc[s], hf.srv_cur_cost[s]); });
}

// price_kernel over L candidate blocks whose values are set (DESIGN.md §3.16, §3.20): threshold and above
// ([L*S*A], device; a NULL above column is not written), the current allocation the fleet's, or with `chain` the
// trace's c_l from its winner blocks ([L*S]).  With acc_count ([L*M*A], device; DESIGN.md §3.25) block l prices at
// row l's AccCount.
void enqueue_price(wva_handle* h, int L, const AllocCols& cand, float* threshold, const AllocCols& above,
                   const AllocCols* chain, const int32_t* acc_count = nullptr) {
    const HostFleet& hf = h->hf;
    const long long warps = (long long)L * hf.S;
    if (warps * hf.A <= 0) return;
    const PriceArgs g{h->df, cand, threshold, above, chain ? *chain : AllocCols{}, L};
    if (acc_count)
        price_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, h->stream>>>(ProfilePriceArgs{g, acc_count});
    else
        price_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, h->stream>>>(g);
    h->launches++;
}

// wva_analyze's sizing and values into cand ([S*A]), then price_kernel: threshold ([S*A], device) and above
// ([S*A] records; at least S, which the sizing's winners use first).
int enqueue_price_thresholds(wva_handle* h, float* threshold, const AllocCols& cand, const AllocCols& above) {
    int rc = enqueue_size(h, cand, &above);
    if (rc) return rc;
    enqueue_price(h, 1, cand, threshold, above, nullptr);
    CK(cudaGetLastError());
    return WVA_OK;
}

// The price threshold grid and trace (DESIGN.md §3.20): wva_workload_grid's or wva_workload_trace's call with
// price_kernel after the winners.  threshold and above's columns are the call's further device columns in d_price,
// copied straight to the caller.  The cost rule is checked per level before any launch; for a trace c_t is known only
// from the winners, so it is checked per tick after the sync, on the winner block's host copy.
//
// With `prof` (the profile price thresholds, DESIGN.md §3.25) the rows also carry acc_cost and perf_* (a NULL
// column: the fleet's own).  The call is then the profile path's (enqueue_profile_trace, in grid mode on a grid),
// price_kernel prices at the rows' AccCount when that column is given, and the cost rule reads the rows'
// perf_present.  With every column NULL it is the workload call's, byte and launch for launch.
int run_price_levels(wva_handle* h, const wva_fleet* fleet, int32_t L, const float* rpm, const int32_t* in,
                     const int32_t* out, const wva_profile_rows* prof, float* threshold, wva_allocs* above,
                     wva_allocs* candidates, wva_allocs* winners, bool trace) {
    if (h && winners && fleet && L > 0 && (long long)fleet->n_servers * fleet->n_acc > 0 && !threshold)
        return h->fail(WVA_ERR_BAD_ARG, "threshold is NULL");
    const char* name = prof ? (trace ? "profile price threshold trace" : "profile price threshold grid")
                            : (trace ? "price threshold trace" : "price threshold grid");
    const uint8_t* present = prof ? prof->perf_present : nullptr;
    const bool rows = prof && (prof->acc_cost || prof->perf_present || prof->perf_alpha || prof->perf_beta ||
                               prof->perf_gamma || prof->perf_delta || prof->perf_acc_count || prof->perf_max_batch ||
                               prof->perf_at_tokens);
    Cols cols(16);
    AllocCols dab{};  // above's device columns, set by place
    LevelMore more;
    more.place = [&](HostCall& c) {
        const HostFleet& hf = h->hf;
        std::string what = price_factor_refusal(hf);
        if (what.empty() && !trace)
            what = price_cost_refusal(hf, L, rpm, in, out, present, "level", [&](int, int s) {
                return std::make_pair(hf.srv_cur_acc[s], hf.srv_cur_cost[s]);
            });
        if (!what.empty()) return h->fail(WVA_ERR_UNSUPPORTED, what.c_str());
        // threshold first, at the buffer's start; then the above columns the caller wants (SIZE_MAX: not placed)
        const size_t n = c.n_cand;
        cols.take(4 * n, threshold);
        Block ab{};
#define PRICE_ABOVE(name, type, required) \
    ab.off.name = above && above->name ? cols.take(sizeof(type) * n, above->name) : SIZE_MAX;
        WVA_ALLOC_COLUMNS(PRICE_ABOVE)
#undef PRICE_ABOVE
        CK(h->d_price.ensure(cols.bytes));
        char* d = (char*)h->d_price.p;
#define PRICE_ABOVE_DEV(name, type, required) dab.name = ab.off.name == SIZE_MAX ? nullptr : (type*)(d + ab.off.name);
        WVA_ALLOC_COLUMNS(PRICE_ABOVE_DEV)
#undef PRICE_ABOVE_DEV
        c.extra = &cols;
        c.extra_dev = d;
        return WVA_OK;
    };
    if (trace)
        more.check = [&](const HostCall& c) {
            const HostFleet& hf = h->hf;
            const uint8_t* feasible = (const uint8_t*)(c.win_host + c.bw.off.feasible);
            const int32_t* acc = (const int32_t*)(c.win_host + c.bw.off.acc);
            const float* cost = (const float*)(c.win_host + c.bw.off.cost);
            // c_t per server, advanced tick by tick as price_cost_refusal walks the rows in order
            std::vector<std::pair<int, float>> cur(hf.S);
            for (int s = 0; s < hf.S; ++s) cur[s] = {hf.srv_cur_acc[s], hf.srv_cur_cost[s]};
            const std::string what = price_cost_refusal(hf, L, rpm, in, out, present, "tick", [&](int t, int s) {
                const std::pair<int, float> ct = cur[s];
                const size_t j = (size_t)t * hf.S + s;
                if (feasible[j]) cur[s] = {acc[j], cost[j]};
                return ct;
            });
            return what.empty() ? WVA_OK : h->fail(WVA_ERR_UNSUPPORTED, what.c_str());
        };
    return run_levels(
        h, fleet, L, name, rpm ? nullptr : "NULL arrival rate list", prof != nullptr, candidates, winners,
        [&](const AllocCols& dc, const AllocCols& dw) {
            const int32_t* acc_count = nullptr;  // row l's AccCount, on the device
            const int rc = rows ? enqueue_profile_trace(h, L, rpm, in, out, *prof, dc, dw, trace, &acc_count)
                                : enqueue_workload(h, L, rpm, in, out, dc, dw, trace);
            if (rc) return rc;
            enqueue_price(h, L, dc, (float*)h->d_price.p, dab, trace ? &dw : nullptr, acc_count);
            CK(cudaGetLastError());
            return WVA_OK;
        },
        more);
}

// ---- SLO bounds: where each load pair's two searches turn nil and stop binding (DESIGN.md §3.18) ----------------
// The load pairs (pairs, batch sizes Ns, sorted by descending N) get one N-entry table each in lg_tabs, as the level
// calls build them.  bounds_tail solves both ends of every pair into the end records, the stored-vector re-run takes
// the items it bailed on, and bounds_kernel writes the entries.  g carries the device columns of the call's buffer
// (ends, out); the launches do not depend on the fleet once it has a load pair.
int enqueue_slo_bounds(wva_handle* h, const std::vector<int>& pairs, const std::vector<int>& Ns,
                       const std::vector<int>& cand_of_pair, BoundsArgs& g) {
    const HostFleet& hf = h->hf;
    int rc = ensure_ctrl(h);
    if (rc) return rc;
    PairTables& pt = h->lg_tabs;
    Cols c(16);
    const size_t o_cop = c.put(cand_of_pair.data(), 4 * cand_of_pair.size());
    rc = upload_tables(h, pt, pairs, Ns, false, c, [](char*) {});
    if (rc) return rc;
    rc = build_tables(h, h->df, pt);
    if (rc) return rc;
    const int n = pt.n;
    FbRun fb;
    rc = prepare_fallback(h, 0, 2 * n, n ? pt.len_max : 0, fb);
    if (rc) return rc;
    set_tables(g, h->df, pt);
    g.cand_of_pair = (const int*)((const char*)pt.lists.p + o_cop);
    g.counter = (unsigned*)h->d_ctrl.p + CTRL_COUNTER;
    g.fb = fb.list;
    CK(cudaEventRecord(h->ev_k0, h->stream));
    if (n > 0) {
        rc = launch_tail(h, bounds_tail, bounds_fallback, g, (2ll * n + 31) / 32, fb);
        if (rc) return rc;
    } else {
        CK(cudaEventRecord(h->ev_k1, h->stream));
    }
    const long long n_out = 2ll * hf.S * hf.A;
    if (n_out > 0) {
        bounds_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, h->stream>>>(g);
        h->launches++;
    }
    CK(cudaGetLastError());
    return WVA_OK;
}

// ---- grid path (K2 + K3) ----------------------------------------------------
int validate_grid(wva_handle* h, const wva_grid* g) {
    if (!g) return h->fail(WVA_ERR_BAD_ARG, "grid is NULL");
    if (g->n_batch < 0 || g->n_replicas < 0) return h->fail(WVA_ERR_BAD_ARG, "negative grid size");
    if ((g->n_batch > 0 && !g->batch) || (g->n_replicas > 0 && !g->replicas))
        return h->fail(WVA_ERR_BAD_ARG, "NULL grid column");
    for (int i = 0; i < g->n_batch; ++i)
        if (g->batch[i] < 1 || g->batch[i] > (1 << 20)) return h->fail(WVA_ERR_BAD_ARG, "batch size out of range");
    for (int i = 0; i < g->n_replicas; ++i)
        if (g->replicas[i] < 1) return h->fail(WVA_ERR_BAD_ARG, "replica count out of range");
    return WVA_OK;
}

struct GridPlan {
    GridArgs args;
    FbRun fb;
    size_t n_cells;
    int Bmax;
    Cols cells{256};  // layout of d_cells; the copy-back goes to the caller's cell table
};

// Per-cell columns kept on the device for every grid solve: flags + ttft/itl/rho (+ throughput
// when the caller asked for it).  They travel to the host only when `cells` names a column.
int ensure_cells(wva_handle* h, GridPlan& plan, const wva_cells* cells) {
    const bool want = cells && (cells->flags || cells->ttft || cells->itl || cells->rho || cells->throughput);
    const wva_cells dst = want ? *cells : wva_cells{};
    const size_t nc = plan.n_cells;
    Cols& c = plan.cells;
    const size_t o_flags = c.take(nc, dst.flags), o_ttft = c.take(4 * nc, dst.ttft), o_itl = c.take(4 * nc, dst.itl),
                 o_rho = c.take(4 * nc, dst.rho), o_thr = c.take(4 * nc, dst.throughput);
    CK(h->d_cells.ensure(c.bytes));
    char* p = (char*)h->d_cells.p;
    plan.args.cells.flags = (uint8_t*)(p + o_flags);
    plan.args.cells.ttft = (float*)(p + o_ttft);
    plan.args.cells.itl = (float*)(p + o_itl);
    plan.args.cells.rho = (float*)(p + o_rho);
    plan.args.cells.throughput = dst.throughput ? (float*)(p + o_thr) : nullptr;
    plan.args.want_cells = want ? 1 : 0;
    return WVA_OK;
}

int prepare_grid(wva_handle* h, const wva_grid* grid, GridPlan* plan) {
    const HostFleet& hf = h->hf;
    const int A = hf.A, S = hf.S, B = grid->n_batch, R = grid->n_replicas;
    const size_t n_pairs = std::max(S * A, 1);
    int Bmax = 1;
    for (int i = 0; i < B; ++i) Bmax = std::max(Bmax, grid->batch[i]);
    // the grid's columns in the lists image: batch[B], batch_rank[B], rank_to_bi[B], replicas[R], then each pair's
    // table offset and index (-1 without a table)
    PairTables& pt = h->grid_tabs;
    Cols c(16);
    const size_t o_lists = c.take(sizeof(int) * (size_t)(3 * B + R)), o_poff = c.take(sizeof(long long) * n_pairs),
                 o_pidx = c.take(sizeof(int) * n_pairs);
    std::vector<int> key(grid->batch, grid->batch + B);
    key.insert(key.end(), grid->replicas, grid->replicas + R);
    key.push_back(B);
    if (!pt.holds(h->epoch_tokens, key)) {
        // shared service-rate tables for every pair that carries load
        std::vector<int> tab_pair;
        for (int s = 0; s < S; ++s)
            for (int a = 0; a < A; ++a)
                if (hf.pair_class(s, a, true) == PAIR_LOAD && hf.srv_out_tokens[s] >= 1) tab_pair.push_back(s * A + a);
        const int n_tab = (int)tab_pair.size();
        if ((long long)n_tab * Bmax > 0xffffffffll) return h->fail(WVA_ERR_UNSUPPORTED, "grid tables above 2^32 entries");
        int rc = upload_tables(h, pt, tab_pair, std::vector<int>(n_tab, Bmax), true, c, [&](char* p) {
            int* lists = (int*)(p + o_lists);
            std::vector<int> order(B);
            std::iota(order.begin(), order.end(), 0);
            std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return grid->batch[x] < grid->batch[y]; });
            for (int i = 0; i < B; ++i) {
                lists[i] = grid->batch[i];
                lists[B + order[i]] = i;      // batch_rank[bi]
                lists[2 * B + i] = order[i];  // rank_to_bi[rank]
            }
            for (int i = 0; i < R; ++i) lists[3 * B + i] = grid->replicas[i];
            long long* pair_off = (long long*)(p + o_poff);
            int* pair_idx = (int*)(p + o_pidx);
            std::fill(pair_off, pair_off + n_pairs, -1ll);
            std::fill(pair_idx, pair_idx + n_pairs, -1);
            for (int t = 0; t < n_tab; ++t) {
                pair_off[tab_pair[t]] = (long long)t * Bmax;
                pair_idx[tab_pair[t]] = t;
            }
        });
        if (rc) return rc;
        pt.epoch = h->epoch_tokens;
        pt.key = std::move(key);
    }
    // every cell of a pair with a table builds the queue model of its batch size
    const int Nmax = pt.n > 0 && B > 0 && R > 0 ? Bmax : 0;
    if (!hf.queue_fits(Nmax))
        return h->fail(WVA_ERR_UNSUPPORTED,
                       "queue model of 2^31 states or more (batch size x (1 + max_queue_to_batch_ratio))");
    // [tables x batch] constants, then the [server x replica] rate block grid_order fills (always allocated)
    CK(h->d_pb.ensure(sizeof(float4) * ((size_t)pt.n * std::max(B, 1) + (size_t)S * std::max(R, 1) + 1)));
    const char* d = (const char*)pt.lists.p;
    GridArgs& g = plan->args;
    g = GridArgs{};
    g.f = h->df;
    g.batch = (const int*)(d + o_lists);
    g.batch_rank = g.batch + B;
    g.rank_to_bi = g.batch + 2 * B;
    g.replicas = g.batch + 3 * B;
    g.B = B;
    g.R = R;
    g.tab = (const double*)pt.tab.p;
    g.ls = (const float*)pt.ls.p;
    g.pair_tab_off = (const long long*)(d + o_poff);
    g.pair_tab_idx = (const int*)(d + o_pidx);
    g.pb = (const float4*)h->d_pb.p;
    g.rt = (float4*)h->d_pb.p + (size_t)pt.n * std::max(B, 1);
    const unsigned long long n_cells = (unsigned long long)S * A * B * R;
    if (n_cells > 0xfffffff0ull) return h->fail(WVA_ERR_UNSUPPORTED, "grid too large for one call (>= 2^32 cells)");
    g.n_cells = (long long)n_cells;
    plan->n_cells = (size_t)n_cells;
    const size_t nc = std::max<size_t>(plan->n_cells, 1);
    // sort workspace: order u32 [n_cells] | items u64 | items_sorted u64 | item counter |
    // per-cell records in global item order (32 x 16 bytes per item) | grid_order's chunk list.
    // A sort chunk (up to kCandChunk candidates of one pair, so at most n_cells / kCandChunk + S*A chunks) ends with
    // at most one partial item.
    const size_t max_chunks = nc / kCandChunk + n_pairs;
    const size_t max_items = (nc + 31) / 32 + max_chunks;
    Cols ws(256);
    const size_t o_order = ws.take(4 * nc), o_items = ws.take(8 * max_items), o_sorted = ws.take(8 * max_items),
                 o_count = ws.take(4 * (2 * kClasses + 32)), o_recs = ws.take(512 * max_items),
                 o_chunks = ws.take(sizeof(uint4) * max_chunks);
    CK(h->d_sort.ensure(ws.bytes));
    char* w = (char*)h->d_sort.p;
    g.order = (unsigned*)(w + o_order);
    g.items = (unsigned long long*)(w + o_items);
    g.items_sorted = (unsigned long long*)(w + o_sorted);
    g.item_count = (unsigned*)(w + o_count);
    g.recs = (uint4*)(w + o_recs);
    g.chunks = (uint4*)(w + o_chunks);
    h->dbg_plan = g.item_count + 2 * kClasses + 1;
    const size_t n_best = std::max<size_t>((size_t)S * A * R, 1);
    CK(h->d_best.ensure(sizeof(int) * n_best));
    g.best_rank = (int*)h->d_best.p;
    const size_t n_pairs_alloc = std::max<size_t>((size_t)S * A, 1);
    Cols rows(256);
    const size_t o_rows = rows.take((2 * sizeof(double) + sizeof(int)) * n_best + 64),  // row_acc | row_sump | row_j
        o_pair_rec = rows.take(48 * n_pairs_alloc), o_grp = rows.take(sizeof(unsigned) * n_best),
                 o_bound = rows.take(sizeof(unsigned long long) * std::max(S, 1)), o_cand = rows.take(sizeof(int4) * n_best);
    CK(h->d_rows.ensure(rows.bytes));
    g.row_acc = (double*)((char*)h->d_rows.p + o_rows);
    g.row_sump = g.row_acc + n_best;
    g.row_j = (int*)(g.row_sump + n_best);
    g.pair_rec = (float4*)((char*)h->d_rows.p + o_pair_rec);
    g.row_grp = (unsigned*)((char*)h->d_rows.p + o_grp);
    g.bound = (unsigned long long*)((char*)h->d_rows.p + o_bound);
    g.row_cand = (int4*)((char*)h->d_rows.p + o_cand);
    // grid_order ranks a server's rows in shared memory, and a cell's key holds the accelerator in 8 bits and the batch
    // size in 24; outside those limits every cell is evaluated (grid_order still walks the shared runs)
    g.prune = A <= 256 && Bmax < (1 << 24) && (long long)A * R <= kOrderMaxRows;
    g.Bmax = Bmax;
    int rc = prepare_fallback(h, 0, (int)std::min<size_t>(nc, (size_t)1 << 22), Nmax, plan->fb);
    if (rc) return rc;
    g.fb_count = plan->fb.list.count;
    g.fb_cells = plan->fb.list.item;
    g.fb_cap = plan->fb.list.cap;
    {
        // grid_kernel's long queue: items of at least ~min_len states, at most long_per_sm per SM
        const int min_len = 1024;
        int long_per_sm = kGkLong;
        if (const char* e = getenv("WVA_GRID_LONG")) long_per_sm = std::min(std::max(atoi(e), -1), kGkWarps / 4);
        g.long_per_sm = long_per_sm;
        g.long_cls = 254 - std::min(std::max((int)(log2f((float)min_len) * 12.0f), 0), 254);
        g.long_cap = (unsigned)(std::max(long_per_sm, 0) * h->sm_count);
        g.n_ctas = h->sm_count;
    }
    if (h->dbg_cycles) {
        CK(h->d_dbg.ensure(sizeof(unsigned) * nc * 2));
        CK(cudaMemsetAsync(h->d_dbg.p, 0, sizeof(unsigned) * nc * 2, h->stream));
        g.dbg_cycles = (unsigned*)h->d_dbg.p;
        g.dbg_n = nc;
        h->dbg_n = nc;
    }
    plan->Bmax = Bmax;
    // the step's first kernel, enqueued after every buffer it or the step uses is in place (a DevBuf that grows frees
    // its old memory)
    return build_tables(h, h->df, pt, g.batch, B, (float4*)h->d_pb.p, g.item_count, kItemCountWords);
}

// timed: record ev_k0 / ev_k1 around grid_kernel for wva_last_kernel_ms, and launch grid_kernel ordinarily.  A record
// of a timing event between two kernels makes the second wait for the first to finish (no programmatic overlap), so
// only calls that read the timing (those with host results) record them.
int enqueue_grid(wva_handle* h, GridPlan& plan, const AllocCols& winners, bool timed) {
    GridArgs& g = plan.args;
    const HostFleet& hf = h->hf;
    int rc = WVA_OK;
    if (timed && plan.n_cells == 0) CK(cudaEventRecord(h->ev_k0, h->stream));
    if (plan.n_cells > 0) {
        if (g.want_cells) g.prune = 0;  // every cell is evaluated and stored
        // the rows; without a cell table the shared-chain cells and each server's bound; the cells left for
        // grid_kernel, then their sort
        const size_t order_smem = (long long)hf.A * g.Bmax <= kOrderTabEntries ? (size_t)hf.A * g.Bmax * 32 : 0;
        rc = launch_pdl(h, grid_order, (unsigned)hf.S, kOrderThreads, order_smem, g);
        const long long cand_smem = cand_stage_bytes(g.B, g.R, g.Bmax);
        if (!rc)
            rc = launch_pdl(h, grid_sort_cands, (unsigned)(kCandCtasPerSm * h->sm_count), kCandThreads,
                            cand_smem <= kCandStageBytes ? (size_t)cand_smem : 0, g);
        if (!rc) rc = launch_pdl(h, grid_items_scatter, (unsigned)(16 * h->sm_count), 256, 0, g);  // warp per item
        if (rc) return rc;
        const size_t smem = (size_t)kGkWarps * kGkWarpD * sizeof(double);
        if (timed) {  // wva_last_kernel_ms = the dominant kernel alone; after the record there is no overlap to gain
            CK(cudaEventRecord(h->ev_k0, h->stream));
            grid_kernel<<<(unsigned)h->sm_count, kGkThreads, smem, h->stream>>>(g);
            h->launches++;
        } else {
            rc = launch_pdl(h, grid_kernel, (unsigned)h->sm_count, kGkThreads, smem, g);
            if (rc) return rc;
        }
    }
    if (timed) CK(cudaEventRecord(h->ev_k1, h->stream));
    if (plan.n_cells > 0) {
        rc = launch_fallback(h, grid_fallback, g, plan.fb, true);
        if (rc) return rc;
        if (g.want_cells) {  // the shared-chain cells with a cell table: one warp per 32 rows and slice of ranks
            const size_t n_warps = ((size_t)hf.S * hf.A * g.R + 31) / 32 * ((size_t)(g.B + kSharedSlice - 1) / kSharedSlice);
            const unsigned ctas = (unsigned)((n_warps + kSharedThreads / 32 - 1) / (kSharedThreads / 32));
            grid_shared<<<ctas, kSharedThreads, 0, h->stream>>>(g);
            h->launches++;
        }
    }
    if (hf.S > 0) {
        rc = launch_pdl(h, grid_finalize, (unsigned)hf.S, 256, 0, g, winners);
        if (rc) return rc;
    }
    CK(cudaGetLastError());
    return WVA_OK;
}


// ---- limited mode: SolveGreedy on the host over device-computed candidates --------------
// pkg/solver/greedy.go:35-341.  The candidate generation (the expensive part) ran on the
// device; the greedy pass is inherently sequential over a shared capacity map (SURVEY.md
// §8e), so it stays on the host.  Sorts are stable (the reference's pdqsort is not): ties
// resolve by server id / accelerator id.
struct GreedyEntry {  // greedy.go:16-22
    int server, priority, cur = 0;
    std::vector<int> accs;  // candidate accelerator ids ordered by value
    float delta = 0.f;
};

inline int cmp_f32(float a, float b) {  // cmp.Compare: NaN sorts first
    const bool an = a != a, bn = b != b;
    if (an || bn) return an && bn ? 0 : (an ? -1 : 1);
    return a < b ? -1 : (a > b ? 1 : 0);
}

class GreedySolver {
  public:
    GreedySolver(const HostFleet& f, std::vector<HostCand>& cand, std::vector<HostCand>& win)
        : f_(f), cand_(cand), win_(win), avail_(f.type_capacity.begin(), f.type_capacity.end()) {}

    void run() {
        const int S = f_.S, A = f_.A;
        std::vector<GreedyEntry> pool;
        pool.reserve(S);
        for (int s = 0; s < S; ++s) {
            win_[s] = HostCand{};
            win_[s].acc = WVA_ACC_NONE;
            GreedyEntry e;
            e.server = s;
            e.priority = f_.srv_priority[s];
            for (int a = 0; a < A; ++a)
                if (at(s, a).feasible) e.accs.push_back(a);
            if (e.accs.empty()) continue;
            std::stable_sort(e.accs.begin(), e.accs.end(),
                             [&](int x, int y) { return cmp_f32(at(s, x).value, at(s, y).value) < 0; });
            e.delta = e.accs.size() > 1 ? at(s, e.accs[1]).value - at(s, e.accs[0]).value : FLT_MAX;
            pool.push_back(std::move(e));
        }
        std::vector<GreedyEntry*> entries;
        for (auto& e : pool) entries.push_back(&e);
        std::stable_sort(entries.begin(), entries.end(),
                         [&](GreedyEntry* x, GreedyEntry* y) { return order(*x, *y) < 0; });
        if (f_.delayed_best_effort) {
            std::vector<GreedyEntry*> un = allocate(entries);
            best_effort(un);
        } else {
            size_t i = 0;
            while (i < entries.size()) {  // makePriorityGroups :321-341
                size_t j = i + 1;
                while (j < entries.size() && entries[j]->priority == entries[i]->priority) ++j;
                std::vector<GreedyEntry*> group(entries.begin() + i, entries.begin() + j);
                std::vector<GreedyEntry*> un = allocate(group);
                best_effort(un);
                i = j;
            }
        }
    }

  private:
    HostCand& at(int s, int a) { return cand_[(size_t)s * f_.A + a]; }
    HostCand& cur(const GreedyEntry& e) { return at(e.server, e.accs[e.cur]); }
    int units(int s, int a) const {
        const int c = f_.perf_acc_count[(size_t)f_.srv_model[s] * f_.A + a];
        return (c <= 0 ? 1 : c) * f_.acc_mult[a];
    }
    int order(GreedyEntry& a, GreedyEntry& b) {  // greedy.go:76-85
        if (a.priority != b.priority) return a.priority < b.priority ? -1 : 1;
        if (a.delta == b.delta) return cmp_f32(cur(b).value, cur(a).value);
        return cmp_f32(b.delta, a.delta);
    }
    std::vector<GreedyEntry*> allocate(std::vector<GreedyEntry*> q) {  // greedy.go:107-166
        std::vector<GreedyEntry*> un;
        size_t head = 0;
        while (head < q.size()) {
            GreedyEntry* top = q[head++];
            if (top->accs.empty()) continue;
            HostCand& al = cur(*top);
            const int g = al.acc;
            if (g < 0 || g >= f_.A) continue;  // accelerator "" (zero-replica allocation)
            const int t = f_.acc_type[g];
            const int count = al.replicas * units(top->server, g);
            if (avail_[t] >= count) {
                avail_[t] -= count;
                win_[top->server] = al;
                continue;
            }
            top->cur++;
            if (top->cur + 1 < (int)top->accs.size()) {
                top->delta = at(top->server, top->accs[top->cur + 1]).value - cur(*top).value;
            } else if (top->cur == (int)top->accs.size()) {
                un.push_back(top);
                continue;
            } else {
                top->delta = FLT_MAX;
            }
            // slices.BinarySearchFunc: leftmost position whose element does not order before top
            auto it = std::partition_point(q.begin() + head, q.end(), [&](GreedyEntry* e) { return order(*e, *top) < 0; });
            q.insert(it, top);
        }
        return un;
    }
    void scale_to(HostCand& al, int replicas) {  // greedy.go:206-211
        const float factor = (float)replicas / (float)al.replicas;
        al.cost *= factor;
        al.value *= factor;
        al.replicas = replicas;
    }
    void allocate_maximally(const std::vector<GreedyEntry*>& es) {  // greedy.go:194-223
        for (GreedyEntry* e : es)
            for (int a : e->accs) {
                HostCand& al = at(e->server, a);
                if (al.acc < 0 || al.acc >= f_.A) continue;
                const int upr = units(e->server, al.acc);
                if (upr <= 0) continue;
                const int t = f_.acc_type[al.acc];
                const int mx = std::min(avail_[t] / upr, al.replicas);
                if (mx > 0) {
                    scale_to(al, mx);
                    win_[e->server] = al;
                    avail_[t] -= mx * upr;
                    break;
                }
            }
    }
    void allocate_equally(const std::vector<GreedyEntry*>& es) {  // greedy.go:239-316
        struct Ticket {
            bool present = true, active = false, allocated = false;
            int type = 0, upr = 0, n = 0;
            HostCand* fin = nullptr;
        };
        std::vector<Ticket> tk(es.size());
        size_t live = es.size();
        while (live > 0) {
            for (size_t k = 0; k < es.size(); ++k) {
                Ticket& t = tk[k];
                if (!t.present) continue;
                if (!t.active) {
                    for (int a : es[k]->accs) {
                        HostCand& al = at(es[k]->server, a);
                        if (al.acc < 0 || al.acc >= f_.A) continue;
                        const int upr = units(es[k]->server, al.acc);
                        if (upr > 0 && avail_[f_.acc_type[al.acc]] >= upr) {
                            t.active = true;
                            t.type = f_.acc_type[al.acc];
                            t.upr = upr;
                            t.fin = &al;
                            break;
                        }
                    }
                    if (!t.active) {
                        t.present = false;
                        --live;
                        continue;
                    }
                }
                if (std::min(avail_[t.type] / t.upr, t.fin->replicas) > 0) {
                    t.n++;
                    avail_[t.type] -= t.upr;
                    t.allocated = true;
                } else {
                    t.present = false;
                    --live;
                }
            }
        }
        for (size_t k = 0; k < es.size(); ++k)
            if (tk[k].allocated) {
                scale_to(*tk[k].fin, tk[k].n);
                win_[es[k]->server] = *tk[k].fin;
            }
    }
    void best_effort(const std::vector<GreedyEntry*>& un) {  // greedy.go:169-190
        switch (f_.saturation_policy) {
        case WVA_SAT_PRIORITY_EXHAUSTIVE: allocate_maximally(un); break;
        case WVA_SAT_PRIORITY_ROUND_ROBIN: {
            size_t i = 0;
            while (i < un.size()) {
                size_t j = i + 1;
                while (j < un.size() && un[j]->priority == un[i]->priority) ++j;
                allocate_equally(std::vector<GreedyEntry*>(un.begin() + i, un.begin() + j));
                i = j;
            }
            break;
        }
        case WVA_SAT_ROUND_ROBIN: allocate_equally(un); break;
        default: break;
        }
    }
    const HostFleet& f_;
    std::vector<HostCand>& cand_;
    std::vector<HostCand>& win_;
    std::vector<int> avail_;
};

void block_to_cands(const void* host_block, const Block& b, std::vector<HostCand>& out) {
    out.resize(b.n);
#define BLOCK_LOAD(name, type, required) \
    for (size_t i = 0; i < b.n; ++i) out[i].name = ((const type*)((const char*)host_block + b.off.name))[i];
    WVA_ALLOC_COLUMNS(BLOCK_LOAD)
#undef BLOCK_LOAD
}
void cands_to_abi(const std::vector<HostCand>& v, wva_allocs* out) {
    if (!out) return;
#define ABI_STORE(name, type, required) \
    if (out->name)                      \
        for (size_t i = 0; i < v.size(); ++i) out->name[i] = v[i].name;
    WVA_ALLOC_COLUMNS(ABI_STORE)
#undef ABI_STORE
}

// The required columns must be there; the others read as 0 when NULL.
bool abi_to_cands(const wva_allocs* in, size_t n, std::vector<HostCand>& out) {
    if (!in) return false;
#define ABI_REQUIRED(name, type, required) \
    if (required && n && !in->name) return false;
    WVA_ALLOC_COLUMNS(ABI_REQUIRED)
#undef ABI_REQUIRED
    out.assign(n, HostCand{});
#define ABI_LOAD(name, type, required) \
    if (in->name)                      \
        for (size_t i = 0; i < n; ++i) out[i].name = in->name[i];
    WVA_ALLOC_COLUMNS(ABI_LOAD)
#undef ABI_LOAD
    return true;
}

// resident analyze + greedy solve with host outputs
int run_greedy_host(wva_handle* h, wva_allocs* candidates, wva_allocs* winners) {
    const HostFleet& hf = h->hf;
    if (!hf.every_acc_typed())
        return h->fail(WVA_ERR_BAD_ARG, "limited mode needs a type id and a capacity for every accelerator");
    HostCall c{(size_t)hf.S * hf.A, true, false};
    const int rc = run_host(h, c, [&](const AllocCols& dc, const AllocCols& dw) {
        return enqueue_size(h, dc, &dw);  // the unlimited kernel also assigns value = transition penalty
    });
    if (rc) return rc;
    std::vector<HostCand> cand, win((size_t)hf.S);
    block_to_cands(c.cand_host, c.bc, cand);
    GreedySolver(hf, cand, win).run();
    cands_to_abi(cand, candidates);
    cands_to_abi(win, winners);
    h->last_win = std::move(win);
    h->last_kind = 2;
    return WVA_OK;
}

}  // namespace

// =============================================================================
// C ABI
// =============================================================================
extern "C" {

void wva_tunables_default(wva_tunables* t) {
    if (!t) return;
    t->max_queue_to_batch_ratio = 10;  // pkg/config/defaults.go:18
    t->accel_penalty_factor = 0.1f;    // pkg/config/defaults.go:21
}

int wva_abi_version(void) { return WVA_ABI_VERSION; }

const char* wva_strerror(int code) {
    switch (code) {
    case WVA_OK: return "ok";
    case WVA_ERR_BAD_ARG: return "bad argument";
    case WVA_ERR_NO_DEVICE: return "no CUDA device";
    case WVA_ERR_CUDA: return "CUDA runtime error";
    case WVA_ERR_NOMEM: return "out of memory";
    case WVA_ERR_STATE: return "call sequence error";
    case WVA_ERR_UNSUPPORTED: return "input outside the supported domain";
    default: return "unknown error";
    }
}

const char* wva_last_error(const wva_handle* h) { return h ? h->err.c_str() : ""; }

int wva_create(wva_handle** out, int device) {
    if (!out) return WVA_ERR_BAD_ARG;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return WVA_ERR_NO_DEVICE;
    if (cudaSetDevice(device) != cudaSuccess) return WVA_ERR_NO_DEVICE;
    wva_handle* h = new (std::nothrow) wva_handle();
    if (!h) return WVA_ERR_NOMEM;
    h->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->sm_count = prop.multiProcessorCount;
    cudaFuncSetAttribute(grid_order, cudaFuncAttributeMaxDynamicSharedMemorySize, kOrderTabEntries * 32);
    cudaFuncSetAttribute(grid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)((size_t)kGkWarps * kGkWarpD * sizeof(double)));
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&h->ev_k0) != cudaSuccess || cudaEventCreate(&h->ev_k1) != cudaSuccess ||
        cudaEventCreate(&h->ev_d0) != cudaSuccess || cudaEventCreate(&h->ev_d1) != cudaSuccess) {
        delete h;
        return WVA_ERR_CUDA;
    }
    *out = h;
    return WVA_OK;
}

void wva_destroy(wva_handle* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->ev_k0) cudaEventDestroy(h->ev_k0);
    if (h->ev_k1) cudaEventDestroy(h->ev_k1);
    if (h->ev_d0) cudaEventDestroy(h->ev_d0);
    if (h->ev_d1) cudaEventDestroy(h->ev_d1);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

// ---------------------------------------------------------------------------
// Winner-block all-gather over peer memory (NVLink / NVSwitch), fused into ONE kernel per step:
// CTA d copies this rank's block into rank d's gathered buffer (slot = this rank) with plain peer
// stores, publishes the step's epoch in rank d's flag word for this rank (release, system scope),
// then waits until rank d's block has arrived HERE.  When the kernel retires every slot of the
// local gathered buffer holds this step's blocks.  Two buffer parities: a fast rank may already
// publish step e+1 while a slow one still reads step e.  The payload is 40 B per server, so the
// exchange is latency: two NVLink hops instead of a library collective's launch + protocol.
// ---------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(256) xchg_publish(const char* __restrict__ src, size_t bytes, char* const* __restrict__ peers,
                                                    int world, int rank, size_t slot_stride, size_t flags_off,
                                                    unsigned long long epoch, int* err) {
    const int d = blockIdx.x;
    const size_t parity_off = (size_t)(epoch & 1ull) * (size_t)world * slot_stride;
    char* dst = peers[d] + parity_off + (size_t)rank * slot_stride;
    const size_t n16 = bytes / 16;
    for (size_t i = threadIdx.x; i < n16; i += blockDim.x) ((int4*)dst)[i] = ((const int4*)src)[i];
    for (size_t i = 16 * n16 + threadIdx.x; i < bytes; i += blockDim.x) dst[i] = src[i];
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        // my flag word in rank d's memory: flags[src rank]
        volatile unsigned long long* theirs = (volatile unsigned long long*)(peers[d] + flags_off) + rank;
        *theirs = epoch;
        __threadfence_system();
        // wait for rank d's block of this epoch in MY memory
        volatile unsigned long long* mine = (volatile unsigned long long*)(peers[rank] + flags_off) + d;
        const long long t0 = clock64();
        while (*mine < epoch) {
            if (clock64() - t0 > (4ll << 30)) {  // ~2 s: a peer is gone; report instead of hanging the GPU
                *err = 1;
                break;
            }
            __nanosleep(200);
        }
        __threadfence_system();
    }
}
}  // namespace

extern "C" {
int wva_xchg_create(wva_handle* h, int world, int rank, size_t block_bytes, void* ipc_handle_out /* 64 bytes */) {
    if (!h || world < 1 || rank < 0 || rank >= world || !ipc_handle_out) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    auto& x = h->xchg;
    x.world = world;
    x.rank = rank;
    x.block_bytes = block_bytes;
    x.slot_stride = (block_bytes + 255) / 256 * 256;
    x.flags_off = 2 * (size_t)world * x.slot_stride;
    x.local_bytes = x.flags_off + 8 * (size_t)world + 256;
    CK(cudaMalloc((void**)&x.local, x.local_bytes));  // its own allocation: IPC exports whole allocations
    CK(cudaMemset(x.local, 0, x.local_bytes));
    CK(cudaMalloc((void**)&x.d_peer, sizeof(char*) * world));
    CK(cudaMalloc((void**)&x.d_err, sizeof(int)));
    CK(cudaMemset(x.d_err, 0, sizeof(int)));
    x.peer.assign(world, nullptr);
    x.peer[rank] = x.local;
    x.epoch = 0;
    cudaIpcMemHandle_t hd;
    CK(cudaIpcGetMemHandle(&hd, x.local));
    static_assert(sizeof(hd) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(ipc_handle_out, &hd, sizeof(hd));
    return WVA_OK;
}
int wva_xchg_open(wva_handle* h, int peer_rank, const void* ipc_handle) {
    if (!h || !ipc_handle || peer_rank < 0 || peer_rank >= h->xchg.world) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    auto& x = h->xchg;
    if (peer_rank != x.rank) {
        cudaIpcMemHandle_t hd;
        memcpy(&hd, ipc_handle, sizeof(hd));
        void* p = nullptr;
        CK(cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
        x.peer[peer_rank] = (char*)p;
    }
    bool all = true;
    for (char* p : x.peer) all = all && p != nullptr;
    if (all) CK(cudaMemcpy(x.d_peer, x.peer.data(), sizeof(char*) * x.world, cudaMemcpyHostToDevice));
    return WVA_OK;
}
// Enqueue the exchange of `src_block` (device memory, block_bytes) on the handle's stream; returns the
// device address of the gathered buffer of this step ([world][slot_stride] bytes) in *gathered.
int wva_xchg_publish(wva_handle* h, const void* src_block, void** gathered, size_t* slot_stride) {
    if (!h || !src_block || h->xchg.world < 1 || !h->xchg.d_peer) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    auto& x = h->xchg;
    for (char* p : x.peer)
        if (!p) return h->fail(WVA_ERR_STATE, "wva_xchg_publish: not every peer buffer is open");
    ++x.epoch;
    xchg_publish<<<x.world, 256, 0, h->stream>>>((const char*)src_block, x.block_bytes, x.d_peer, x.world, x.rank, x.slot_stride,
                                                 x.flags_off, x.epoch, x.d_err);
    h->launches++;
    if (gathered) *gathered = x.local + (size_t)(x.epoch & 1ull) * (size_t)x.world * x.slot_stride;
    if (slot_stride) *slot_stride = x.slot_stride;
    CK(cudaGetLastError());
    return WVA_OK;
}
int wva_xchg_error(wva_handle* h) {  // after a synchronize: 1 = a peer never arrived
    if (!h || !h->xchg.d_err) return 0;
    int e = 0;
    cudaMemcpy(&e, h->xchg.d_err, sizeof(int), cudaMemcpyDeviceToHost);
    return e;
}
int wva_xchg_destroy(wva_handle* h) {
    if (!h) return WVA_ERR_BAD_ARG;
    auto& x = h->xchg;
    cudaSetDevice(h->device);
    for (int r = 0; r < (int)x.peer.size(); ++r)
        if (r != x.rank && x.peer[r]) cudaIpcCloseMemHandle(x.peer[r]);
    if (x.local) cudaFree(x.local);
    if (x.d_peer) cudaFree(x.d_peer);
    if (x.d_err) cudaFree(x.d_err);
    x = wva_handle::Xchg();
    return WVA_OK;
}
}  // extern "C"

void* wva_stream(wva_handle* h) { return h ? (void*)h->stream : nullptr; }

int wva_synchronize(wva_handle* h) {
    if (!h) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    return WVA_OK;
}

int64_t wva_launch_count(const wva_handle* h) { return h ? h->launches : 0; }
float wva_last_kernel_ms(const wva_handle* h) { return h ? h->last_kernel_ms : 0.f; }
float wva_last_device_ms(const wva_handle* h) { return h ? h->last_device_ms : 0.f; }

int wva_upload(wva_handle* h, const wva_fleet* fleet) {
    if (!h) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    CK(cudaStreamSynchronize(h->stream));
    return WVA_OK;
}

int wva_update_load(wva_handle* h, const float* arrival_rpm, const int32_t* in_tokens, const int32_t* out_tokens) {
    if (!h) return WVA_ERR_BAD_ARG;
    if (!h->resident) return h->fail(WVA_ERR_STATE, "no resident fleet (call wva_upload first)");
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));  // the pinned stage may still feed an earlier async copy
    HostFleet& hf = h->hf;
    const size_t S = hf.S;
    bool tokens_changed = false, class_changed = false;
    if (arrival_rpm) {
        for (size_t s = 0; s < S && !class_changed; ++s)
            class_changed = ((arrival_rpm[s] == 0.0f) != (hf.srv_arrival_rpm[s] == 0.0f)) ||
                            ((arrival_rpm[s] < 0.0f) != (hf.srv_arrival_rpm[s] < 0.0f));
        hf.srv_arrival_rpm.assign(arrival_rpm, arrival_rpm + S);
        memcpy((char*)h->stage.p + h->col_rate.off, arrival_rpm, 4 * S);
    }
    if (in_tokens) {
        tokens_changed = tokens_changed || !std::equal(in_tokens, in_tokens + S, hf.srv_in_tokens.begin());
        hf.srv_in_tokens.assign(in_tokens, in_tokens + S);
        memcpy((char*)h->stage.p + h->col_in.off, in_tokens, 4 * S);
    }
    if (out_tokens) {
        tokens_changed = tokens_changed || !std::equal(out_tokens, out_tokens + S, hf.srv_out_tokens.begin());
        hf.srv_out_tokens.assign(out_tokens, out_tokens + S);
        memcpy((char*)h->stage.p + h->col_out.off, out_tokens, 4 * S);
    }
    // the three load columns are adjacent in the arena: one copy
    const size_t lo = h->col_rate.off, hi = h->col_out.off + h->col_out.bytes;
    if (S) CK(cudaMemcpyAsync((char*)h->arena.p + lo, (char*)h->stage.p + lo, hi - lo, cudaMemcpyHostToDevice, h->stream));
    if (tokens_changed || class_changed) h->epoch_tokens++;
    h->last_kind = 0;
    return WVA_OK;
}

int wva_analyze(wva_handle* h, const wva_fleet* fleet, wva_allocs* candidates) {
    if (!h || !candidates) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    // Server.Calculate also assigns value = transition penalty: run the unlimited
    // kernel into a scratch winner block so that candidate values are final
    wva_allocs dummy{};
    return run_size_host(h, candidates, &dummy);
}

// SolveGreedy + best-effort policies over a candidate table the caller already holds (host only, no device work):
// the multi-GPU limited mode all-gathers the per-shard candidate tables and runs this redundantly on every rank.
int wva_solve_greedy(const wva_fleet* fleet, wva_allocs* candidates, wva_allocs* winners) {
    if (fleet_problem(fleet) || !winners) return WVA_ERR_BAD_ARG;
    HostFleet hf;
    fill_host_fleet(hf, fleet);
    if (!hf.every_acc_typed()) return WVA_ERR_BAD_ARG;
    std::vector<HostCand> cand, win((size_t)hf.S);
    if (!abi_to_cands(candidates, (size_t)hf.S * hf.A, cand)) return WVA_ERR_BAD_ARG;
    GreedySolver(hf, cand, win).run();
    cands_to_abi(cand, candidates);
    cands_to_abi(win, winners);
    return WVA_OK;
}

int wva_resolve(wva_handle* h, wva_allocs* candidates, wva_allocs* winners) {
    if (!h || !winners) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    if (!h->resident) return h->fail(WVA_ERR_STATE, "no resident fleet (call wva_upload first)");
    if (!h->hf.unlimited) return run_greedy_host(h, candidates, winners);
    const int rc = run_size_host(h, candidates, winners);
    if (rc == WVA_OK) h->last_kind = 1;
    return rc;
}

int wva_solve(wva_handle* h, const wva_fleet* fleet, wva_allocs* candidates, wva_allocs* winners) {
    if (!h || !winners) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    return wva_resolve(h, candidates, winners);
}

int wva_resolve_device(wva_handle* h, wva_allocs* winners_dev) {
    if (!h || !winners_dev) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    if (!h->resident) return h->fail(WVA_ERR_STATE, "no resident fleet (call wva_upload first)");
    if (!h->hf.unlimited) return h->fail(WVA_ERR_UNSUPPORTED, "limited (greedy) mode has host outputs only: use wva_resolve");
    const HostFleet& hf = h->hf;
    const Block bc = block_layout((size_t)hf.S * hf.A);
    CK(h->d_cand_block.ensure(bc.bytes + 16));
    const AllocCols dc = block_cols(h->d_cand_block.p, bc);
    const AllocCols dw = cols_from_abi(winners_dev);
    CK(cudaEventRecord(h->ev_d0, h->stream));
    int rc = enqueue_size(h, dc, &dw);
    if (rc) return rc;
    CK(cudaEventRecord(h->ev_d1, h->stream));
    return WVA_OK;
}

int wva_grid_solve_device(wva_handle* h, const wva_grid* grid, wva_allocs* winners_dev) {
    if (!h || !winners_dev) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    if (!h->resident) return h->fail(WVA_ERR_STATE, "no resident fleet (call wva_upload first)");
    int rc = validate_grid(h, grid);
    if (rc) return rc;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    GridPlan plan;
    rc = prepare_grid(h, grid, &plan);
    if (rc) return rc;
    rc = ensure_cells(h, plan, nullptr);
    if (rc) return rc;
    // untimed: nothing reads the timing events after a call without host results
    return enqueue_grid(h, plan, cols_from_abi(winners_dev), false);
}

int wva_grid_solve(wva_handle* h, const wva_fleet* fleet, const wva_grid* grid, wva_cells* cells, wva_allocs* winners) {
    if (!h || !winners) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    int rc = validate_grid(h, grid);
    if (rc) return rc;
    rc = upload_fleet(h, fleet);
    if (rc) return rc;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    GridPlan plan;
    rc = prepare_grid(h, grid, &plan);
    if (rc) return rc;
    rc = ensure_cells(h, plan, cells);
    if (rc) return rc;
    if (plan.args.want_cells && plan.n_cells)  // cells that are never analysed must read back as 0
        CK(cudaMemsetAsync(h->d_cells.p, 0, plan.cells.bytes, h->stream));
    HostCall c{0, false, true, &plan.cells, h->d_cells.p};
    rc = run_host(h, c, [&](const AllocCols&, const AllocCols& dw) { return enqueue_grid(h, plan, dw, true); });
    if (rc) return rc;
    scatter_block(c.win_host, c.bw, winners);
    h->last_kind = 1;
    return WVA_OK;
}

int wva_size_grid(wva_handle* h, const wva_fleet* fleet, int32_t n_batch, const int32_t* batch, wva_allocs* candidates,
                  wva_allocs* winners) {
    if (!h || !winners) return WVA_ERR_BAD_ARG;
    if (n_batch < 0 || (n_batch > 0 && !batch)) return h->fail(WVA_ERR_BAD_ARG, "negative batch count or NULL batch list");
    for (int i = 0; i < n_batch; ++i)
        if (batch[i] < 1 || batch[i] > (1 << 20)) return h->fail(WVA_ERR_BAD_ARG, "batch size out of range");
    if (const char* what = fleet_problem(fleet)) return h->fail(WVA_ERR_BAD_ARG, what);
    if ((long long)fleet->n_servers * fleet->n_acc * n_batch >= (1ll << 31))
        return h->fail(WVA_ERR_UNSUPPORTED, "size grid too large for one call (>= 2^31 candidates)");
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    HostCall c{(size_t)fleet->n_servers * fleet->n_acc * n_batch, candidates != nullptr, true};
    rc = run_host(h, c, [&](const AllocCols& dc, const AllocCols& dw) {
        return enqueue_size_grid(h, n_batch, batch, dc, dw);
    });
    if (rc) return rc;
    scatter_block(c.cand_host, c.bc, candidates);
    scatter_block(c.win_host, c.bw, winners);
    h->last_kind = 1;
    return WVA_OK;
}

int wva_load_grid(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                  wva_allocs* candidates, wva_allocs* winners) {
    if (h && winners && (n_levels < 0 || (n_levels > 0 && !arrival_rpm)))
        return h->fail(WVA_ERR_BAD_ARG, "negative level count or NULL level list");
    return run_levels(h, fleet, n_levels, "load grid", nullptr, false, candidates, winners,
                      [&](const AllocCols& dc, const AllocCols& dw) {
                          return enqueue_load_grid(h, n_levels, arrival_rpm, dc, dw);
                      });
}

int wva_slo_grid(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* slo_itl,
                 const float* slo_ttft, const float* slo_tps, wva_allocs* candidates, wva_allocs* winners) {
    const char* null_rows = !slo_itl || !slo_ttft || !slo_tps ? "NULL target row list" : nullptr;
    return run_levels(h, fleet, n_levels, "SLO grid", null_rows, false, candidates, winners,
                      [&](const AllocCols& dc, const AllocCols& dw) {
                          return enqueue_slo_grid(h, n_levels, slo_itl, slo_ttft, slo_tps, dc, dw);
                      });
}

int wva_workload_grid(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                      const int32_t* in_tokens, const int32_t* out_tokens, wva_allocs* candidates,
                      wva_allocs* winners) {
    const char* null_rows = !arrival_rpm || !in_tokens || !out_tokens ? "NULL row list" : nullptr;
    return run_levels(h, fleet, n_levels, "workload grid", null_rows, false, candidates, winners,
                      [&](const AllocCols& dc, const AllocCols& dw) {
                          return enqueue_workload(h, n_levels, arrival_rpm, in_tokens, out_tokens, dc, dw, false);
                      });
}

int wva_workload_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks, const float* arrival_rpm,
                       const int32_t* in_tokens, const int32_t* out_tokens, wva_allocs* candidates,
                       wva_allocs* winners) {
    const char* null_rows = !arrival_rpm || !in_tokens || !out_tokens ? "NULL row list" : nullptr;
    return run_levels(h, fleet, n_ticks, "workload trace", null_rows, false, candidates, winners,
                      [&](const AllocCols& dc, const AllocCols& dw) {
                          return enqueue_workload(h, n_ticks, arrival_rpm, in_tokens, out_tokens, dc, dw, true);
                      });
}

int wva_slo_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks, const float* arrival_rpm,
                  const int32_t* in_tokens, const int32_t* out_tokens, const float* slo_itl, const float* slo_ttft,
                  const float* slo_tps, wva_allocs* candidates, wva_allocs* winners) {
    return run_levels(h, fleet, n_ticks, "SLO trace", nullptr, false, candidates, winners,
                      [&](const AllocCols& dc, const AllocCols& dw) {
                          return enqueue_slo_trace(h, n_ticks, arrival_rpm, in_tokens, out_tokens, slo_itl, slo_ttft,
                                                   slo_tps, dc, dw);
                      });
}

int wva_profile_grid(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const wva_profile_rows* rows,
                     wva_allocs* candidates, wva_allocs* winners) {
    const wva_profile_rows own{};
    return run_levels(h, fleet, n_levels, "profile grid", nullptr, true, candidates, winners,
                      [&](const AllocCols& dc, const AllocCols& dw) {
                          return enqueue_profile_grid(h, n_levels, rows ? *rows : own, dc, dw);
                      });
}

int wva_profile_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks, const float* arrival_rpm,
                      const int32_t* in_tokens, const int32_t* out_tokens, const wva_profile_rows* rows,
                      wva_allocs* candidates, wva_allocs* winners) {
    const wva_profile_rows own{};
    return run_levels(h, fleet, n_ticks, "profile trace", nullptr, true, candidates, winners,
                      [&](const AllocCols& dc, const AllocCols& dw) {
                          return enqueue_profile_trace(h, n_ticks, arrival_rpm, in_tokens, out_tokens,
                                                       rows ? *rows : own, dc, dw);
                      });
}

int wva_load_intervals(wva_handle* h, const wva_fleet* fleet, const float* rpm_lo, const float* rpm_hi,
                       wva_intervals* out) {
    if (!h) return WVA_ERR_BAD_ARG;
    if (!out) return h->fail(WVA_ERR_BAD_ARG, "out is NULL");
    if (const char* what = fleet_problem(fleet)) return h->fail(WVA_ERR_BAD_ARG, what);
    const int S = fleet->n_servers, M = out->max_per_server;
    if (M < 1) return h->fail(WVA_ERR_BAD_ARG, "max_per_server below 1");
    if (S > 0 && (!rpm_lo || !rpm_hi || !out->count || !out->truncated || !out->start_rpm))
        return h->fail(WVA_ERR_BAD_ARG, "NULL bound or output column");
    if ((long long)S * M >= (1ll << 31))
        return h->fail(WVA_ERR_UNSUPPORTED, "load intervals too large for one call (>= 2^31 records)");
    for (int s = 0; s < S; ++s)
        if (!std::isfinite(rpm_lo[s]) || !std::isfinite(rpm_hi[s]) || rpm_lo[s] < 0.0f || !(rpm_lo[s] <= rpm_hi[s]))
            return h->fail(WVA_ERR_BAD_ARG, "bound NaN, infinite or negative, or rpm_lo above rpm_hi");
    Cols cols(16);
    const size_t o_count = cols.take(4 * (size_t)S, out->count), o_trunc = cols.take((size_t)S, out->truncated),
                 o_start = cols.take(4 * (size_t)S * M, out->start_rpm);
    return run_walk(h, fleet, cols, (size_t)S * M, true, {&out->rec},
                    [&](const WalkArgs& w, char* d, size_t rec_bytes) {
                        IntervalArgs g{w};
                        g.M = M;
                        g.count = (int*)(d + o_count);
                        g.truncated = (uint8_t*)(d + o_trunc);
                        g.start = (float*)(d + o_start);
                        return enqueue_load_intervals(h, rpm_lo, rpm_hi, g, rec_bytes);
                    });
}

int wva_load_margins(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                     const float* rpm_lo, const float* rpm_hi, wva_margins* out) {
    return load_margins_call(h, fleet, n_levels, arrival_rpm, nullptr, nullptr, false, nullptr, nullptr, rpm_lo, rpm_hi,
                             out, false);
}

int wva_load_margin_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks, const float* arrival_rpm,
                          const float* rpm_lo, const float* rpm_hi, wva_margins* out) {
    return load_margins_call(h, fleet, n_ticks, arrival_rpm, nullptr, nullptr, false, nullptr, nullptr, rpm_lo, rpm_hi,
                             out, true);
}

int wva_workload_margins(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                         const int32_t* in_tokens, const int32_t* out_tokens, const float* rpm_lo, const float* rpm_hi,
                         wva_margins* out) {
    return load_margins_call(h, fleet, n_levels, arrival_rpm, in_tokens, out_tokens, true, nullptr, nullptr, rpm_lo,
                             rpm_hi, out, false);
}

int wva_workload_margin_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks, const float* arrival_rpm,
                              const int32_t* in_tokens, const int32_t* out_tokens, const float* rpm_lo,
                              const float* rpm_hi, wva_margins* out) {
    return load_margins_call(h, fleet, n_ticks, arrival_rpm, in_tokens, out_tokens, true, nullptr, nullptr, rpm_lo,
                             rpm_hi, out, true);
}

int wva_profile_margins(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                        const int32_t* in_tokens, const int32_t* out_tokens, const wva_profile_rows* rows,
                        const float* rpm_lo, const float* rpm_hi, wva_margins* out) {
    const wva_profile_rows own{};
    return load_margins_call(h, fleet, n_levels, arrival_rpm, in_tokens, out_tokens, true, rows ? rows : &own, nullptr,
                             rpm_lo, rpm_hi, out, false);
}

int wva_profile_margin_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks, const float* arrival_rpm,
                             const int32_t* in_tokens, const int32_t* out_tokens, const wva_profile_rows* rows,
                             const float* rpm_lo, const float* rpm_hi, wva_margins* out) {
    const wva_profile_rows own{};
    return load_margins_call(h, fleet, n_ticks, arrival_rpm, in_tokens, out_tokens, true, rows ? rows : &own, nullptr,
                             rpm_lo, rpm_hi, out, true);
}

int wva_slo_margins(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                    const int32_t* in_tokens, const int32_t* out_tokens, const float* slo_itl, const float* slo_ttft,
                    const float* slo_tps, const float* rpm_lo, const float* rpm_hi, wva_margins* out) {
    const TargetRows slo{slo_itl, slo_ttft, slo_tps};
    return load_margins_call(h, fleet, n_levels, arrival_rpm, in_tokens, out_tokens, true, nullptr, &slo, rpm_lo,
                             rpm_hi, out, false);
}

int wva_slo_margin_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks, const float* arrival_rpm,
                         const int32_t* in_tokens, const int32_t* out_tokens, const float* slo_itl,
                         const float* slo_ttft, const float* slo_tps, const float* rpm_lo, const float* rpm_hi,
                         wva_margins* out) {
    const TargetRows slo{slo_itl, slo_ttft, slo_tps};
    return load_margins_call(h, fleet, n_ticks, arrival_rpm, in_tokens, out_tokens, true, nullptr, &slo, rpm_lo,
                             rpm_hi, out, true);
}

int wva_price_thresholds(wva_handle* h, const wva_fleet* fleet, float* threshold, wva_allocs* above,
                         wva_allocs* candidates) {
    if (!h) return WVA_ERR_BAD_ARG;
    if (const char* what = fleet_problem(fleet)) return h->fail(WVA_ERR_BAD_ARG, what);
    const long long n = (long long)fleet->n_servers * fleet->n_acc;
    if (n > 0 && !threshold) return h->fail(WVA_ERR_BAD_ARG, "threshold is NULL");
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    const std::string what = price_refusal(h->hf);
    if (!what.empty()) return h->fail(WVA_ERR_UNSUPPORTED, what.c_str());
    Cols th(16);
    th.take(4 * (size_t)n, threshold);
    CK(h->d_price.ensure(th.bytes));
    HostCall c{(size_t)n, candidates != nullptr, above != nullptr && n > 0, &th, h->d_price.p};
    c.win_blocks = (size_t)std::max(fleet->n_acc, 1);  // above, and the sizing's S winners before it
    rc = run_host(h, c, [&](const AllocCols& dc, const AllocCols& dw) {
        return enqueue_price_thresholds(h, (float*)h->d_price.p, dc, dw);
    });
    // no single solution to summarise (upload_fleet cleared last_kind)
    if (rc) return rc;
    scatter_block(c.cand_host, c.bc, candidates);
    if (c.win_host) scatter_block(c.win_host, c.bw, above);
    return WVA_OK;
}

int wva_price_threshold_grid(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                             const int32_t* in_tokens, const int32_t* out_tokens, float* threshold, wva_allocs* above,
                             wva_allocs* candidates, wva_allocs* winners) {
    return run_price_levels(h, fleet, n_levels, arrival_rpm, in_tokens, out_tokens, nullptr, threshold, above,
                            candidates, winners, false);
}

int wva_price_threshold_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks, const float* arrival_rpm,
                              const int32_t* in_tokens, const int32_t* out_tokens, float* threshold, wva_allocs* above,
                              wva_allocs* candidates, wva_allocs* winners) {
    return run_price_levels(h, fleet, n_ticks, arrival_rpm, in_tokens, out_tokens, nullptr, threshold, above,
                            candidates, winners, true);
}

int wva_profile_price_threshold_grid(wva_handle* h, const wva_fleet* fleet, int32_t n_levels, const float* arrival_rpm,
                                     const int32_t* in_tokens, const int32_t* out_tokens, const wva_profile_rows* rows,
                                     float* threshold, wva_allocs* above, wva_allocs* candidates,
                                     wva_allocs* winners) {
    const wva_profile_rows own{};
    return run_price_levels(h, fleet, n_levels, arrival_rpm, in_tokens, out_tokens, rows ? rows : &own, threshold,
                            above, candidates, winners, false);
}

int wva_profile_price_threshold_trace(wva_handle* h, const wva_fleet* fleet, int32_t n_ticks,
                                      const float* arrival_rpm, const int32_t* in_tokens, const int32_t* out_tokens,
                                      const wva_profile_rows* rows, float* threshold, wva_allocs* above,
                                      wva_allocs* candidates, wva_allocs* winners) {
    const wva_profile_rows own{};
    return run_price_levels(h, fleet, n_ticks, arrival_rpm, in_tokens, out_tokens, rows ? rows : &own, threshold,
                            above, candidates, winners, true);
}

int wva_slo_bounds(wva_handle* h, const wva_fleet* fleet, wva_slo_bounds_out* out) {
    if (!h) return WVA_ERR_BAD_ARG;
    if (const char* what = fleet_problem(fleet)) return h->fail(WVA_ERR_BAD_ARG, what);
    if (!out) return h->fail(WVA_ERR_BAD_ARG, "out is NULL");
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    const HostFleet& hf = h->hf;
    std::vector<int> pairs, Ns;
    rc = sorted_pairs(h, hf, [&](int s, int a) { return hf.pair_class(s, a, true) == PAIR_LOAD; }, pairs, Ns);
    if (rc) return rc;
    const size_t n = pairs.size(), n_out = 2 * (size_t)hf.S * hf.A;
    std::vector<int> cand_of_pair((size_t)hf.S * hf.A, -1);
    for (size_t e = 0; e < n; ++e) cand_of_pair[pairs[e]] = (int)e;
    // the end records (their feasible column comes back to name a pair whose solve failed), then the entries
    std::vector<uint8_t> solved(2 * n, 1);
    Cols b(16);
    const size_t o_solved = b.take(2 * n, solved.data()), o_ttft = b.take(8 * n), o_itl = b.take(8 * n);
    const size_t o_kind = b.take(n_out, out->kind), o_ylo = b.take(4 * n_out, out->y_lo),
                 o_yhi = b.take(4 * n_out, out->y_hi), o_b1 = b.take(4 * n_out, out->b1),
                 o_b2 = b.take(4 * n_out, out->b2);
    CK(h->d_bounds.ensure(b.bytes));
    char* d = (char*)h->d_bounds.p;
    BoundsArgs g{};
    g.ends.feasible = (uint8_t*)(d + o_solved);
    g.ends.ttft = (float*)(d + o_ttft);
    g.ends.itl = (float*)(d + o_itl);
    g.out = BoundsOut{(uint8_t*)(d + o_kind), (float*)(d + o_ylo), (float*)(d + o_yhi), (float*)(d + o_b1),
                      (float*)(d + o_b2)};
    HostCall c{0, false, false, &b, d};
    rc = run_host(h, c, [&](const AllocCols&, const AllocCols&) {
        return enqueue_slo_bounds(h, pairs, Ns, cand_of_pair, g);
    });
    // no single solution to summarise (upload_fleet cleared last_kind)
    if (rc == WVA_ERR_UNSUPPORTED)
        for (size_t i = 0; i < 2 * n; ++i)
            if (solved[i] == 0) {
                const int s = pairs[i / 2] / hf.A, a = pairs[i / 2] % hf.A;
                const std::string what = "boundary solve at lambda_" + std::string(i % 2 ? "max" : "min") +
                                         " of server " + std::to_string(s) + ", accelerator " + std::to_string(a) +
                                         ": input outside the supported numeric domain (rescale loop does not "
                                         "terminate)";
                return h->fail(WVA_ERR_UNSUPPORTED, what.c_str());
            }
    return rc;
}

// System.AllocateByType + CreateAllocationDiff over the most recent solution (include/wva_b200.h).
int wva_summarize(wva_handle* h, wva_summary* out) {
    if (!h || !out) return WVA_ERR_BAD_ARG;
    CK(cudaSetDevice(h->device));
    if (!h->resident || h->last_kind == 0) return h->fail(WVA_ERR_STATE, "no solution to summarise (solve first)");
    const HostFleet& hf = h->hf;
    const size_t S = hf.S, T = hf.T;
    if (h->last_kind == 2) {  // greedy winners live on the host: same loops as the kernel
        for (size_t t = 0; t < T; ++t) {
            if (out->type_present) out->type_present[t] = 0;
            if (out->type_count) out->type_count[t] = 0;
            if (out->type_limit) out->type_limit[t] = hf.type_capacity[t];
            if (out->type_cost) out->type_cost[t] = 0.0f;
        }
        std::vector<float> cost(T, 0.0f);
        std::vector<int64_t> cnt(T, 0);
        for (size_t s = 0; s < S; ++s) {
            const HostCand& w = h->last_win[s];
            const int feas = w.feasible, acc = w.acc, rep = w.replicas;
            const float c = w.cost;
            const int m = hf.srv_model[s];
            if (feas && acc >= 0 && acc < hf.A && m >= 0 && m < hf.M) {
                const int t = hf.acc_type[acc];
                if (t >= 0 && t < hf.T) {
                    int inst = 0;
                    if (hf.perf_present[(size_t)m * hf.A + acc]) {
                        inst = hf.perf_acc_count[(size_t)m * hf.A + acc];
                        if (inst <= 0) inst = 1;
                    }
                    cnt[t] += (int64_t)rep * inst * (int64_t)hf.acc_mult[acc];
                    cost[t] = cost[t] + c;
                    if (out->type_present) out->type_present[t] = 1;
                }
            }
            if (out->diff_old_acc) out->diff_old_acc[s] = hf.srv_cur_acc[s];
            if (out->diff_old_replicas) out->diff_old_replicas[s] = hf.srv_cur_replicas[s];
            if (out->diff_new_acc) out->diff_new_acc[s] = feas ? acc : WVA_ACC_ABSENT;
            if (out->diff_new_replicas) out->diff_new_replicas[s] = feas ? rep : 0;
            if (out->diff_cost) out->diff_cost[s] = (feas ? c : 0.0f) - hf.srv_cur_cost[s];
        }
        for (size_t t = 0; t < T; ++t) {
            if (out->type_count) out->type_count[t] = cnt[t];
            if (out->type_cost) out->type_cost[t] = cost[t];
        }
        return WVA_OK;
    }
    if (T > (size_t)kSumMaxTypes) return h->fail(WVA_ERR_UNSUPPORTED, "more accelerator types than summary_kernel owns");
    // device winner block of the last solve
    const Block bw = block_layout(S);
    const AllocCols dw = block_cols(h->d_win_block.p, bw);
    Cols sc(16);
    const size_t o_cnt = sc.take(8 * T, out->type_count), o_pres = sc.take(T, out->type_present),
                 o_lim = sc.take(4 * T, out->type_limit), o_cost = sc.take(4 * T, out->type_cost);
    const size_t o_oa = sc.take(4 * S, out->diff_old_acc), o_na = sc.take(4 * S, out->diff_new_acc),
                 o_or = sc.take(4 * S, out->diff_old_replicas), o_nr = sc.take(4 * S, out->diff_new_replicas),
                 o_dc = sc.take(4 * S, out->diff_cost);
    CK(h->d_summary.ensure(sc.bytes));
    CK(h->out_stage.ensure(sc.bytes));
    char* d = (char*)h->d_summary.p;
    SummaryOut so;
    so.type_count = (long long*)(d + o_cnt);
    so.type_present = (uint8_t*)(d + o_pres);
    so.type_limit = (int*)(d + o_lim);
    so.type_cost = (float*)(d + o_cost);
    so.diff_old_acc = (int*)(d + o_oa);
    so.diff_new_acc = (int*)(d + o_na);
    so.diff_old_replicas = (int*)(d + o_or);
    so.diff_new_replicas = (int*)(d + o_nr);
    so.diff_cost = (float*)(d + o_dc);
    summary_kernel<<<1, 256, 0, h->stream>>>(h->df, dw, so);
    h->launches++;
    CK(cudaGetLastError());
    char* hs = (char*)h->out_stage.p;
    CK(cudaMemcpyAsync(hs, d, sc.bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    sc.scatter(hs);
    return WVA_OK;
}

// MM1KModel.Solve for n triples (include/wva_b200.h).
int wva_mm1k_solve(wva_handle* h, int32_t n, const int32_t* K, const float* lambda, const float* mu, wva_mm1k_out* out) {
    if (!h || !out || n < 0 || (n > 0 && (!K || !lambda || !mu))) return WVA_ERR_BAD_ARG;
    if (n == 0) return WVA_OK;
    for (int i = 0; i < n; ++i)
        if (K[i] < 0) return h->fail(WVA_ERR_BAD_ARG, "MM1K: negative K");  // NewMM1KModel returns nil (mm1kmodel.go:20-22)
    for (int i = 0; i < n; ++i)  // one thread walks the K + 1 states of a triple: bound the launch
        if (K[i] > (1 << 20)) return h->fail(WVA_ERR_UNSUPPORTED, "MM1K: K above 2^20");
    CK(cudaSetDevice(h->device));
    const size_t N = (size_t)n;
    Cols mc(16);
    const size_t i_K = mc.take(4 * N), i_lam = mc.take(4 * N), i_mu = mc.take(4 * N);
    const size_t in_bytes = mc.bytes;
    const size_t o_sum = mc.take(8 * N, out->sum_p), o_valid = mc.take(N, out->is_valid), o_rho = mc.take(4 * N, out->rho),
                 o_nsys = mc.take(4 * N, out->avg_num_in_system), o_thr = mc.take(4 * N, out->throughput),
                 o_resp = mc.take(4 * N, out->avg_resp_time), o_serv = mc.take(4 * N, out->avg_serv_time),
                 o_wait = mc.take(4 * N, out->avg_wait_time), o_qlen = mc.take(4 * N, out->avg_queue_length);
    CK(h->d_summary.ensure(mc.bytes));
    CK(h->out_stage.ensure(mc.bytes));
    char* d = (char*)h->d_summary.p;
    char* hs = (char*)h->out_stage.p;
    memcpy(hs + i_K, K, 4 * N);
    memcpy(hs + i_lam, lambda, 4 * N);
    memcpy(hs + i_mu, mu, 4 * N);
    CK(cudaMemcpyAsync(d, hs, in_bytes, cudaMemcpyHostToDevice, h->stream));
    Mm1kArgs g;
    g.n = n;
    g.K = (const int*)(d + i_K);
    g.lambda = (const float*)(d + i_lam);
    g.mu = (const float*)(d + i_mu);
    g.sum_p = (double*)(d + o_sum);
    g.is_valid = (uint8_t*)(d + o_valid);
    g.rho = (float*)(d + o_rho);
    g.avg_num_in_system = (float*)(d + o_nsys);
    g.throughput = (float*)(d + o_thr);
    g.avg_resp_time = (float*)(d + o_resp);
    g.avg_serv_time = (float*)(d + o_serv);
    g.avg_wait_time = (float*)(d + o_wait);
    g.avg_queue_length = (float*)(d + o_qlen);
    mm1k_kernel<<<(unsigned)((N + 127) / 128), 128, 0, h->stream>>>(g);
    h->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(hs + in_bytes, d + in_bytes, mc.bytes - in_bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    mc.scatter(hs);
    return WVA_OK;
}

int wva_sweep(wva_handle* h, const wva_fleet* fleet, int32_t n_rates, wva_sweep_out* out) {
    if (!h || !out || n_rates < 1) return WVA_ERR_BAD_ARG;
    if (!out->valid || !out->rate || !out->ttft || !out->itl || !out->throughput || !out->rho)
        return h->fail(WVA_ERR_BAD_ARG, "NULL sweep output column");
    CK(cudaSetDevice(h->device));
    int rc = upload_fleet(h, fleet);
    if (rc) return rc;
    rc = ensure_ctrl(h);
    if (rc) return rc;
    const HostFleet& hf = h->hf;
    const int A = hf.A, S = hf.S;
    // every (server, acc) with a profile, ignoring keepAccelerator
    std::vector<int> pairs, lens;
    rc = sorted_pairs(h, hf,
                      [&](int s, int a) {
                          const int m = hf.srv_model[s];
                          return hf.srv_in_tokens[s] >= 0 && hf.srv_out_tokens[s] >= 1 && m >= 0 && m < hf.M &&
                                 hf.perf_present[(size_t)m * A + a];
                      },
                      pairs, lens);
    if (rc) return rc;
    const int n = (int)pairs.size();
    const size_t n_out = (size_t)S * A * n_rates;
    Cols sw(256);
    const size_t o_valid = sw.take(n_out, out->valid), o_rate = sw.take(4 * n_out, out->rate),
                 o_ttft = sw.take(4 * n_out, out->ttft), o_itl = sw.take(4 * n_out, out->itl),
                 o_thr = sw.take(4 * n_out, out->throughput), o_rho = sw.take(4 * n_out, out->rho);
    CK(h->d_sweep.ensure(sw.bytes));
    char* p = (char*)h->d_sweep.p;
    CK(cudaMemsetAsync(p, 0, sw.bytes, h->stream));
    HostCall call{0, false, false, &sw, p};
    call.win_blocks = 0;
    return run_host(h, call, [&](const AllocCols&, const AllocCols&) {
        if (!n) {
            CK(cudaEventRecord(h->ev_k0, h->stream));
            CK(cudaEventRecord(h->ev_k1, h->stream));
            return WVA_OK;
        }
        // the grid's tables, without the ls column: a sweep holds no device memory of its own for them
        PairTables& pt = h->grid_tabs;
        Cols c(16);
        int rc = upload_tables(h, pt, pairs, lens, false, c, [](char*) {});
        if (rc) return rc;
        rc = build_tables(h, h->df, pt);
        if (rc) return rc;
        FbRun fb;
        rc = prepare_fallback(h, 0, (int)std::min<size_t>((size_t)n * n_rates, (size_t)1 << 22), lens[0], fb);
        if (rc) return rc;
        SweepArgs g{};
        g.f = h->df;
        g.pair_list = pt.pair();
        g.pair_N = pt.len();
        g.tab_off = pt.off();
        g.tab = (const double*)pt.tab.p;
        g.n_pairs = n;
        g.n_rates = n_rates;
        g.n_chunks = (n_rates + 31) / 32;
        g.counter = (unsigned*)h->d_ctrl.p + CTRL_COUNTER;
        g.valid = (uint8_t*)(p + o_valid);
        g.rate = (float*)(p + o_rate);
        g.ttft = (float*)(p + o_ttft);
        g.itl = (float*)(p + o_itl);
        g.throughput = (float*)(p + o_thr);
        g.rho = (float*)(p + o_rho);
        g.fb = fb.list;
        CK(cudaEventRecord(h->ev_k0, h->stream));
        // one warp per (pair, chunk) item; the points whose chain left the streaming solve's window are re-run with
        // the stored vector, as the reference
        rc = launch_tail(h, sweep_kernel, sweep_fallback, g, (long long)((unsigned)n * g.n_chunks), fb);
        if (rc) return rc;
        CK(cudaGetLastError());
        return WVA_OK;
    });
}

// ---- self-check of the exact-division primitive (not part of the public ABI) ------------------
// Compares div_recip (Markstein correction around a double-word reciprocal) with div.rn.f64 on
// pseudo-random operands drawn from the solver's exponent windows, including adversarial
// divisors next to powers of two and float32-valued divisors, and div_rate / step_rate (no
// correction) on float32-valued divisors, random and at the least distance a quotient by a
// float32 can have from a rounding midpoint.  Returns the mismatch count.
__global__ void div_selfcheck_kernel(unsigned long long seed, int iters, unsigned long long* mismatches) {
    unsigned long long x = seed ^ (0x9E3779B97F4A7C15ull * (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x + 1));
    auto next = [&]() {  // xorshift64*
        x ^= x >> 12; x ^= x << 25; x ^= x >> 27;
        return x * 0x2545F4914F6CDD1Dull;
    };
    unsigned long long bad = 0;
    for (int it = 0; it < iters; ++it) {
        const unsigned long long r0 = next(), r1 = next(), r2 = next();
        // divisor: mantissa random / float32-valued / all-ones / one-above-power-of-two; exponent in [-60, 60]
        unsigned long long mb = r0 & 0x000FFFFFFFFFFFFFull;
        switch (r2 & 3) {
        case 0: mb &= 0x000FFFFFE0000000ull; break;                 // float32-valued (24-bit significand)
        case 1: mb = 0x000FFFFFFFFFFFFFull - (r0 & 0xff); break;    // just below a power of two
        case 2: mb = r0 & 0xff; break;                              // just above a power of two
        default: break;
        }
        const long long eb = (long long)((r2 >> 8) % 121) - 60;
        const double b = __longlong_as_double((long long)(((unsigned long long)(1023 + eb) << 52) | mb));
        // dividend: random mantissa (sometimes all ones), exponent in [-340, 940] (p * lambda)
        unsigned long long ma = r1 & 0x000FFFFFFFFFFFFFull;
        if (((r2 >> 20) & 7) == 0) ma = 0x000FFFFFFFFFFFFFull - (r1 & 0xf);
        const long long ea = (long long)((r2 >> 24) % 1281) - 340;
        const double a = __longlong_as_double((long long)(((unsigned long long)(1023 + ea) << 52) | ma));
        const Recip rc = make_recip(b);
        const double q = div_recip(a, rc), want = __ddiv_rn(a, b);
        if (__double_as_longlong(q) != __double_as_longlong(want)) ++bad;
        // the cheaper low word used for the normalising sum (zl = RN(e * zh))
        Recip z = rc;
        z.yl = __dmul_rn(__fma_rn(-b, rc.yh, 1.0), rc.yh);
        const double q2 = div_recip(a, z);
        if (__double_as_longlong(q2) != __double_as_longlong(want)) ++bad;
        // division by a service rate (div_rate, no Markstein correction): a float32 divisor drawn as case 0 above
        const float bf = (float)__longlong_as_double((long long)(((unsigned long long)(1023 + eb) << 52) |
                                                                 (r0 & 0x000FFFFFE0000000ull)));
        const RateRecip rr = make_rate_recip(bf);
        if (__double_as_longlong(div_rate(a, rr)) != __double_as_longlong(__ddiv_rn(a, (double)bf))) ++bad;
        // the tail step with the pre-multiplied low word (step_rate): p in [2^-280, 2^880), float32 lambda in
        // [2^-60, 2^60]
        {
            const unsigned long long r3 = next();
            const long long ep = (long long)(r3 % 1160) - 280;
            const double pp = __longlong_as_double((long long)(((unsigned long long)(1023 + ep) << 52) | ma));
            const long long el = (long long)((r3 >> 12) % 121) - 60;
            const double lam = __longlong_as_double(
                (long long)(((unsigned long long)(1023 + el) << 52) | ((r3 >> 20) & 0x000FFFFFE0000000ull)));
            const double got = step_rate(pp, lam, __dmul_rn(lam, rr.yl), rr);
            const double want3 = __ddiv_rn(__dmul_rn(pp, lam), (double)bf);
            if (__double_as_longlong(got) != __double_as_longlong(want3)) ++bad;
        }
        // the hardest float32 divisors: b = M * 2^eb with M odd (24 bits) and a = A * 2^ea with
        // A * 2^25 = M * O -+ 1 for an odd 54-bit O, so that a / b lies 2^-25 / M (~2^-78 relative) from the
        // rounding midpoint O * 2^-25 (scaled); checked through div_rate and through step_rate with lambda a power
        // of two (p = a / lambda exactly)
        {
            const unsigned long long r6 = next(), r7 = next();
            const unsigned M = 0x800001u | ((unsigned)r6 & 0x7FFFFEu);  // odd, in [2^23, 2^24)
            unsigned inv = M;  // M^-1 mod 2^25 by Newton's iteration (each step doubles the correct low bits)
            for (int k = 0; k < 5; ++k) inv *= 2u - M * inv;
            const bool plus = (r6 >> 24) & 1;  // A * 2^25 = M * O + 1 (O = -M^-1) or M * O - 1 (O = M^-1)
            const unsigned long long olo = (plus ? (0u - inv) : inv) & 0x1FFFFFFu;
            const unsigned long long ohi = (1ull << 28) | ((r6 >> 25) & 0xFFFFFFFull);  // O = ohi * 2^25 + olo
            const unsigned long long mlo = (unsigned long long)M * olo;                // < 2^49
            const unsigned long long A = (unsigned long long)M * ohi + ((plus ? mlo + 1 : mlo - 1) >> 25);
            const long long ebh = (long long)(r7 % 120) - 60, eah = (long long)((r7 >> 8) % 1281) - 340;
            const float bh = (float)ldexp((double)M, (int)ebh - 23);
            const double ah = ldexp((double)A, (int)eah - 52);
            const RateRecip rh = make_rate_recip(bh);
            const double wanth = __ddiv_rn(ah, (double)bh);
            if (__double_as_longlong(div_rate(ah, rh)) != __double_as_longlong(wanth)) ++bad;
            const long long elh = (long long)((r7 >> 20) % 121) - 60;
            const long long eph = eah - elh;  // p = a / lambda, kept inside [2^-280, 2^880)
            if (eph >= -279 && eph < 880) {  // A in [2^51, 2^53): p in [2^(eph - 1), 2^(eph + 1))
                const double lam = ldexp(1.0, (int)elh), pp = ldexp((double)A, (int)eph - 52);
                if (__double_as_longlong(step_rate(pp, lam, __dmul_rn(lam, rh.yl), rh)) != __double_as_longlong(wanth)) ++bad;
            }
        }
        // the division by the normalising sum: sum in [1, 2^900), p in [max(2^-280, sum * 2^-960), sum]
        {
            const unsigned long long r4 = next(), r5 = next();
            const long long es = (long long)(r4 % 900);
            const double S = __longlong_as_double((long long)(((unsigned long long)(1023 + es) << 52) | (r5 & 0x000FFFFFFFFFFFFFull)));
            const long long lo = es - 959 > -280 ? es - 959 : -280;
            const long long epp = lo + (long long)((r4 >> 16) % (unsigned long long)(es - lo + 1));
            const double pp = __longlong_as_double((long long)(((unsigned long long)(1023 + epp) << 52) | mb));
            Recip zz;
            zz.b = S;
            zz.yh = __ddiv_rn(1.0, S);
            zz.yl = __dmul_rn(__fma_rn(-S, zz.yh, 1.0), zz.yh);
            const double got = div_recip(pp, zz), want4 = __ddiv_rn(pp, S);
            if (__double_as_longlong(got) != __double_as_longlong(want4)) ++bad;
        }
    }
    if (bad) atomicAdd(mismatches, bad);
}

// ---- diagnostics (not part of the public ABI) ------------------------------------------
// Per-cell SM cycles of the last grid solve, in launch order, followed by the cell ids.
// Runs blocks*256*iters rounds of the checks above; returns the number of results that differ from div.rn.f64.
long long wva_dbg_div_selfcheck(wva_handle* h, unsigned long long seed, int blocks, int iters) {
    if (!h) return -1;
    cudaSetDevice(h->device);
    unsigned long long* d = nullptr;
    if (cudaMalloc(&d, sizeof(unsigned long long)) != cudaSuccess) return -1;
    cudaMemsetAsync(d, 0, sizeof(unsigned long long), h->stream);
    div_selfcheck_kernel<<<blocks, 256, 0, h->stream>>>(seed, iters, d);
    unsigned long long out = ~0ull;
    cudaMemcpyAsync(&out, d, sizeof(out), cudaMemcpyDeviceToHost, h->stream);
    cudaStreamSynchronize(h->stream);
    cudaFree(d);
    return (long long)out;
}

int wva_dbg_read_plan(wva_handle* h, unsigned* out32) {  // grid_items_plan's queue plan: item_count[2*kClasses+1 ..+31]
    if (!h || !h->d_sort.p || !h->dbg_plan) return -1;
    return (int)cudaMemcpy(out32, h->dbg_plan, sizeof(unsigned) * 31, cudaMemcpyDeviceToHost);
}
int wva_dbg_enable_cycles(wva_handle* h, int on) {
    if (!h) return WVA_ERR_BAD_ARG;
    h->dbg_cycles = on != 0;
    return WVA_OK;
}
long long wva_dbg_read_cycles(wva_handle* h, unsigned* cycles, unsigned* cells, long long cap) {
    if (!h || !h->d_dbg.p) return 0;
    const long long n = std::min<long long>((long long)h->dbg_n, cap);
    cudaMemcpy(cycles, h->d_dbg.p, sizeof(unsigned) * n, cudaMemcpyDeviceToHost);
    cudaMemcpy(cells, (unsigned*)h->d_dbg.p + h->dbg_n, sizeof(unsigned) * n, cudaMemcpyDeviceToHost);
    return n;
}

}  // extern "C"

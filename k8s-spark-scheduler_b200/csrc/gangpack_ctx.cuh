// gangpack_ctx.cuh -- private to libgangpack: the context (gp_ctx) with its device buffers, status blocks and CUDA-graph
// cache, and what more than one translation unit of csrc/ shares.  The functions and kernels declared here are defined in
// the .cu file named above them; a helper that one file uses stays static there.
#pragma once

#include "gangpack.h"
#include "gangpack_held.cuh"
#include "gangpack_kernels.cuh"

#include <cstddef>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

using namespace gp;

// Device memory owned by the context: freed when the context is deleted.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    // reserve() for state the kernels leave zeroed after every use: a new allocation starts out all zero
    cudaError_t reserve_zeroed(size_t bytes, cudaStream_t st) {
        if (bytes <= cap) return cudaSuccess;
        const cudaError_t e = reserve(bytes);
        return e != cudaSuccess ? e : cudaMemsetAsync(p, 0, cap, st);
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// n elements of T at an offset of an Arena
template <typename T> struct Piece {
    size_t off, n;
    Piece part(size_t first, size_t count) const { return {off + sizeof(T) * first, count}; }   // elements [first, first + count)
};

// One staging layout in one DevBuf, enqueued on one stream: take() every piece (256-byte-aligned offsets), then reserve()
// once.  The first CUDA error of a helper is kept and every later helper does nothing: the entry calls check() (or sync())
// before its first launch and before it reads anything back.  A piece of 0 elements issues no copy or memset.
struct Arena {
    DevBuf& buf;
    cudaStream_t st;
    size_t size = 0;
    cudaError_t err = cudaSuccess;
    const char* op = nullptr;                    // the helper that met err

    template <typename T> Piece<T> take(size_t n) {
        const Piece<T> p{size, n};
        size += (sizeof(T) * n + 255) & ~(size_t)255;
        return p;
    }
    void reserve() { if (!err) keep(buf.reserve(size), "reserve"); }
    template <typename T> T* ptr(Piece<T> p) const { return reinterpret_cast<T*>(buf.as<char>() + p.off); }
    // the device copy of `host`, or NULL when host is NULL (an absent optional column).  U differs from T only in name
    // (int64_t columns staged as the kernels' long long).
    template <typename T, typename U> T* put(Piece<T> p, const U* host) {
        static_assert(sizeof(T) == sizeof(U), "a piece is uploaded from elements of its own size");
        if (!host) return nullptr;
        if (!err && p.n) keep(cudaMemcpyAsync(ptr(p), host, sizeof(T) * p.n, cudaMemcpyHostToDevice, st), "upload");
        return ptr(p);
    }
    template <typename T, typename U> T* put_or_zero(Piece<T> p, const U* host) { return host ? put(p, host) : zero(p); }
    template <typename T> T* fill(Piece<T> p, int byte) { return fill(p, p, byte); }
    template <typename T> T* zero(Piece<T> p) { return fill(p, p, 0); }
    // one memset over the pieces first .. last (taken in that order) and the padding between them
    template <typename T, typename U> T* fill(Piece<T> first, Piece<U> last, int byte) {
        const size_t bytes = last.off + sizeof(U) * last.n - first.off;
        if (!err && bytes) keep(cudaMemsetAsync(ptr(first), byte, bytes, st), "memset");
        return ptr(first);
    }
    // n elements of device memory to `host`; nothing when host is NULL or n is 0
    template <typename U, typename T> void get(U* host, const T* dev, size_t n) {
        static_assert(sizeof(T) == sizeof(U), "a piece is downloaded into elements of its own size");
        if (!err && host && n) keep(cudaMemcpyAsync(host, dev, sizeof(T) * n, cudaMemcpyDeviceToHost, st), "download");
    }
    template <typename U, typename T> void get(U* host, Piece<T> p) { get(host, ptr(p), p.n); }
    gp_status check(gp_ctx* c) const;
    gp_status sync(gp_ctx* c) { if (!err) keep(cudaStreamSynchronize(st), "synchronise"); return check(c); }

private:
    void keep(cudaError_t e, const char* what) { if (e != cudaSuccess) { err = e; op = what; } }
};

// A status word's bit family decoded by refuse(): the first entry of a table, in table order, whose bits are set
struct Refusal { int bits; gp_status status; const char* what; };

// A fixed sequence of kernel launches / memsets that repeats with identical arguments (one Predicate after the other:
// same buffers, same batch shape) is captured ONCE into a CUDA graph and replayed with a single launch call -- the
// pipelined host path is bound by how fast the host thread can issue its calls, not by the GPU.  The key is the byte image
// of every argument of the sequence; it is captured when the same key is seen twice in a row.
struct GraphCache {
    cudaGraphExec_t exec = nullptr;
    std::vector<char> key, last_key;
    int launches = 0;
    ~GraphCache() { reset(); }
    void reset() { if (exec) cudaGraphExecDestroy(exec); exec = nullptr; key.clear(); last_key.clear(); }
};

static constexpr int32_t kChunkApps = 50000;        // apps per pipelined chunk of gp_pack_batch (~1.5 MB H2D)
static constexpr int32_t kZeroCopyOutApps = 8192;  // batches up to this size write results straight into mapped host memory
static constexpr int kMaxChunks = 16;

// The head of the per-call status block: what gp_last_stats copies to the host
struct StatusHead {
    int err;                                // kErr* bits
    unsigned long long stats[4];            // nodes_scanned, drivers_tried, scan_path_apps, scan_path_nodes (device atomics)
};
static_assert(offsetof(StatusHead, stats) % 8 == 0, "64-bit atomics on the statistics need 8-byte alignment");
static_assert(sizeof(StatusHead) == 40, "gp_last_stats copies the error bits and the four statistics");

// Device status words of one pack call, zeroed by pack_begin or by gp_decide_tables' first classify tile
struct DevStatus {
    StatusHead head;
    unsigned int az_listed, az_claim;       // gp_pack_az_fallback: length of its application list, its claim counter
    unsigned int fifo_cursor;               // FIFO kernels: instance-group cursor
    unsigned int next_app[kMaxChunks];      // per pipelined chunk: application claim counter
    unsigned int spare[3];
};
static_assert(sizeof(DevStatus) == 4 * kStatusWords, "gp_decide_tables zeroes the whole block");

// Pinned host block: the mirror of StatusHead (gp_last_stats) and the error word the kernels write through its mapping
struct PinnedStatus { StatusHead head; volatile int err_word; };

#define GP_CUDA(ctx, expr)                                                                     \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            (ctx)->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                   \
            return GP_ERR_CUDA;                                                                \
        }                                                                                      \
    } while (0)

#define GP_TRY(expr)                                                                           \
    do {                                                                                       \
        const gp_status _s = (expr);                                                           \
        if (_s != GP_OK) return _s;                                                            \
    } while (0)

#include "gangpack_resident.cuh"

struct gp_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    static constexpr int kLanes = 3;       // H2D / kernels / D2H of consecutive chunks overlap across lanes
    cudaStream_t lane[kLanes] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev[kMaxChunks][3] = {};    // per chunk: prep start, pack start, pack end
    cudaEvent_t ev_ready = nullptr, ev_done[kLanes] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_t0 = nullptr;           // GANGPACK_TRACE=2: start of the pipelined batch (timeline of the chunks on stderr)
    int ev_chunks = 0;
    std::string err;

    // snapshot
    Held held;
    int32_t n_nodes = 0, n_groups = 0, n_exec = 0, n_drv = 0, n_slots = 0;
    DevBuf node_cpu, node_mem, node_gpu;        // node-table order (as given)
    DevBuf exec_off, drv_off, exec_order, drv_order;
    DevBuf pair, pair32, sgpu, slot_node, node_slot, drv_slot, groups, snap_flags;
    DevBuf drv_pos;                             // node -> driver-order position, scattered by the layout (gp_build_slots_exec)
    DevBuf snap_part;                           // SnapPart per CTA of gp_build_slots_exec
    DevBuf seg_pre;                             // [n_groups + 1] table segments before each group (gp_build_slots_drv)

    // batch staging; a_rows: the six quantity rows in one pitched block (pack_batch_impl)
    DevBuf a_rows, a_count, a_group, a_skip, a_off;
    DevBuf prep, r_driver, r_exec, scratch, dev_misc, gmin, sortbuf, usagebuf;
    void* pinned_misc = nullptr;                  // PinnedStatus
    DevStatus* status() const { return dev_misc.as<DevStatus>(); }
    PinnedStatus* host_status() const { return static_cast<PinnedStatus*>(pinned_misc); }
    std::vector<int64_t> host_off;
    std::vector<int32_t> eff_seg;                 // gp_packing_efficiency_groups: seg_off [G + 1], then the bucketed nodes
    // gp_set_snapshot's host copy of the layout (Held::host_copy), kept for the az-aware order checks: v_owner[v] (group,
    // roles) and v_pos[v] / v_pos[n_nodes + v] (position of v in its group's executor / driver order)
    std::vector<int32_t> v_owner, v_pos;
    std::vector<uint8_t> v_seen_e, v_seen_d;
    std::vector<int32_t> v_zone_next;             // az-aware order check: next position per zone group
    std::vector<ZoneFifoGroup> zone_groups;       // zone FIFO: per instance group its zones, queue range and scratch rows
    std::vector<int32_t> zone_queue;              // zone FIFO: application indices by instance group (stable counting sort)
    int az_fallback_ctas_per_sm = 0;              // occupancy of gp_pack_az_fallback (queried once)
    std::vector<std::pair<const char*, size_t>> pinned_blocks;   // gp_alloc_pinned allocations (device-mapped under UVA)
    void* one_block = nullptr;                    // gp_pack_one staging (mapped pinned)
    size_t one_bytes = 0;
    int zero_copy = 1;                            // GANGPACK_ZERO_COPY=0 disables reading/writing mapped host buffers in kernels
    int use_tables = 1;                           // GANGPACK_TABLES=0: every independent decision takes the node-order scan
    int fifo_warp = 1;                            // GANGPACK_FIFO_WARP=0: every FIFO application is decided by the whole CTA
    bool async_snapshot = false;                  // gp_config.flags & GP_CFG_ASYNC_SNAPSHOT
    int chunk_apps = kChunkApps;                  // GANGPACK_CHUNK_APPS
    int trace = 0;                                // GANGPACK_TRACE=1: host-side phase timing on stderr
    int pack_ctas_per_sm = 0;                       // occupancy of gp_pack_independent<2> on this device
    int tab_ctas_per_sm[2][2] = {{0, 0}, {0, 0}};   // occupancy of gp_pack_listed<ALGO, OUT>
    int dec_ctas_per_sm[2][2] = {{0, 0}, {0, 0}};   // occupancy of gp_decide_tables<ALGO, OUT>
    // per pipeline lane: shape hash + header, capacity tables, group totals, placement prefixes, per-application shape slot
    struct TableSet { DevBuf hdr, table, total, place, app_slot; } tabs[kLanes];
    bool record_events = true;                    // CUDA events around the kernels (gp_last_stats); the pipelined host path skips them
    bool ev_prep = false;                         // the last pack recorded a prep interval ev[i][0] .. ev[i][1] (not the tables path)
    int use_graphs = 1;                           // GANGPACK_GRAPHS=0: always issue the launches one by one
    GraphCache g_chunk[kMaxChunks + 1];           // per pipelined chunk (+1: an unchunked batch on the context's own stream): classify .. scan
    GraphCache g_snapshot;                        // slot layout of gp_set_snapshot
    DevBuf off_dev;                               // ExecutorNodes offsets derived on the device
    DevBuf fifo_list;                             // FIFO modes: per-instance-group application lists (queue order)
    DevBuf sched, zonebuf, fbview;                // SchedulableResources [3][n_nodes]; staging of the zone entry points;
                                                  // the az-aware fallback's orders and gather view
    DevBuf zoneprep;                              // gp_prepare_cluster_zones*: the undivided orders (Held::orders) and scratch
    // The own scratch of one call of gp_reschedule_executors, gp_reschedule_from_reservations, gp_exceeds_cluster_capacity*,
    // gp_match_node_affinity, gp_reconcile_find_nodes or gp_node_overhead: no state points into it, and the next call's
    // use is ordered after this one's kernels on the context's stream
    DevBuf callbuf;
    // gp_placement_metrics[_device]: staging and scratch of one call; the two words of PmState (zeroed at the start of every
    // call); the host form's records before its refusal check; the dynamic shared memory its kernels may take (0 until the
    // first call on this device)
    DevBuf metricbuf, metricstate;
    std::vector<gp_placement_record> pm_records;
    int pm_smem_limit = 0;
    bool sort_attr_set = false;
    bool recon_attr_set = false;                  // dynamic shared-memory opt-in of gp_sort_tiles<ReconKey> done on this device
    bool fifo_attr_set[2] = {false, false};       // dynamic shared-memory opt-in of gp_pack_fifo_cta<ALGO,*> done on this device

    // the resident tables (gangpack_resident.cuh); each is read by its own entries and those named below, and changed only by
    // its own reset and update
    struct OverheadTable : ResidentTable<gp_overhead_table_size> {   // gangpack_overhead_table.cu; the columns hold the RR flags
        using ResidentTable::ResidentTable;
        DevBuf set[2];                            // member set: set[cur] is live, the other the target of the next rehash
        int cur = 0;
        uint32_t cells = 0;                       // cells of set[cur], a power of two
        long long keys = 0, used = 0;             // live keys; cells holding a key or a tombstone
    } oht{"no overhead table (gp_overhead_table_reset first)"};
    // gangpack_reservation_table.cu, read by the *_resident entries: node id [n_slots], cpu / mem / gpu [3][n_slots]
    ResidentTable<gp_reservation_table_size> rt{"no reservation table (gp_reservation_table_reset first)"};
    // gangpack_label_table.cu, read by the *_resident affinity entries: count, key, val, val_int and val_int_ok
    ResidentTable<gp_label_table_size> lt{"no label table (gp_label_table_reset first)"};
    // gangpack_node_table.cu, read by the *_node_table entries: present, alloc [3], unschedulable, ready, name_key, name_rank
    struct NodeTable : ResidentTable<gp_node_table_size> {
        using ResidentTable::ResidentTable;
        DevBuf gather;                            // the columns one *_node_table call gathers, and its scratch
    } nt{"no node table (gp_node_table_reset first)"};
    // gangpack_driver_table.cu, read by the *_driver_table entries: present, exact, creation, scheduler, group, quantities [6],
    // count, affinity
    struct DriverTable : ResidentTable<gp_driver_table_size> {
        using ResidentTable::ResidentTable;
        DevBuf queue;                             // the queue one *_driver_table call selects, orders and packs, and its scratch
        bool sort_attr_set = false;               // dynamic shared-memory opt-in of gp_sort_tiles<QueueKey> done on this device
    } dt{"no driver table (gp_driver_table_reset first)"};

    gp_stats last{};
};

gp_status fail(gp_ctx* ctx, gp_status st, const std::string& msg);
static inline gp_status fail(gp_ctx* c, gp_status st, const char* who, const char* what) {
    return fail(c, st, std::string(who) + ": " + what);
}

// The prologue of the C ABI entries that enqueue device work: false for a NULL context; takes the tail (into *tail if given)
static inline bool enter(gp_ctx* c, const void** tail = nullptr) {
    const void* t = c ? c->held.take_tail() : nullptr;
    if (tail) *tail = t;
    return c != nullptr;
}

// GP_OK when the requirements are met, otherwise the first one's refusal as `who: what`
static inline gp_status require(gp_ctx* c, Need n, const char* who) { return n.status == GP_OK ? GP_OK : fail(c, n.status, who, n.what); }
static inline gp_status require(gp_ctx* c, Need a, Need b, const char* who) { return a.status != GP_OK ? require(c, a, who) : require(c, b, who); }

inline gp_status Arena::check(gp_ctx* c) const {
    if (!err) return GP_OK;
    c->err = std::string("staging ") + op + ": " + cudaGetErrorString(err);
    return GP_ERR_CUDA;
}

// `who: what` of the first entry of `table` whose bits are set in `word`; GP_OK when there is none
template <size_t K>
static gp_status refuse(gp_ctx* c, int word, const Refusal (&table)[K], const char* who) {
    for (const Refusal& r : table)
        if (word & r.bits) return fail(c, r.status, who, r.what);
    return GP_OK;
}

// Launch kernel k on st; with early, as a programmatic dependent of the kernel before it on st (pdl_wait, pdl_trigger).
template <class... P, class... A>
static cudaError_t launch_pdl(bool early, dim3 grid, dim3 block, cudaStream_t st, void (*k)(P...), A&&... args) {
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = early ? 1 : 0;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, k, std::forward<A>(args)...);
}

// issue(): enqueues the sequence on `st` and returns (status, launches).  See GraphCache.
template <class F>
static gp_status run_cached(gp_ctx* c, GraphCache& gc, const void* key, size_t kn, cudaStream_t st, F&& issue) {
    const char* kb = static_cast<const char*>(key);
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (!c->use_graphs || cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
        cudaGetLastError();
        int n = 0;
        gp_status s = issue(n);
        c->last.kernel_launches += n;
        return s;
    }
    if (gc.exec && gc.key.size() == kn && std::memcmp(gc.key.data(), kb, kn) == 0) {
        GP_CUDA(c, cudaGraphLaunch(gc.exec, st));
        c->last.kernel_launches += gc.launches;
        return GP_OK;
    }
    if (gc.last_key.size() == kn && std::memcmp(gc.last_key.data(), kb, kn) == 0 &&
        cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed) == cudaSuccess) {
        int n = 0;
        const gp_status s = issue(n);
        cudaGraph_t g = nullptr;
        const cudaError_t e = cudaStreamEndCapture(st, &g);
        if (s == GP_OK && e == cudaSuccess && g) {
            cudaGraphExec_t ex = nullptr;
            if (cudaGraphInstantiate(&ex, g, 0) == cudaSuccess) {
                if (gc.exec) cudaGraphExecDestroy(gc.exec);
                gc.exec = ex; gc.key.assign(kb, kb + kn); gc.launches = n;
                cudaGraphDestroy(g);
                GP_CUDA(c, cudaGraphLaunch(gc.exec, st));
                c->last.kernel_launches += n;
                return GP_OK;
            }
        }
        if (g) cudaGraphDestroy(g);
        cudaGetLastError();                 // capture did not work out: issue directly below
        if (s != GP_OK) return s;
    } else {
        cudaGetLastError();
    }
    gc.last_key.assign(kb, kb + kn);
    int n = 0;
    gp_status s = issue(n);
    c->last.kernel_launches += n;
    return s;
}

// ---- gangpack_api.cu -------------------------------------------------------------------------------------------------

// gp_multi_copy's jobs: up to 8 host->device copies in one launch
struct CopyJob { const void* src; void* dst; unsigned long long bytes; };
struct CopyJobs { CopyJob j[8]; int n; };
__global__ void gp_multi_copy(CopyJobs jobs);
__global__ void gp_fill_pair32(int32_t n_slots, const longlong2* __restrict__ pair, SnapMeta* __restrict__ meta,
                               uint2* __restrict__ pair32);
__global__ void gp_scatter_slots(int32_t n_slots, const longlong2* __restrict__ pair, const int64_t* __restrict__ sgpu,
                                 const int32_t* __restrict__ slot_node,
                                 int64_t* __restrict__ cpu, int64_t* __restrict__ mem, int64_t* __restrict__ gpu);

const void* mapped_ptr(gp_ctx* c, const void* p, size_t bytes);
Snapshot make_snapshot(const gp_ctx* c);
gp_status build_snapshot_device(gp_ctx* c, const gp_nodes* dn, int32_t n_exec, int32_t n_drv, cudaStream_t st,
                                bool copy_nodes = false);

// ---- gangpack_pack.cu ------------------------------------------------------------------------------------------------

constexpr int kPrepThreads = 256;
__global__ void gp_prep_apps(int32_t n_apps, AppColumns cols, const uint8_t* __restrict__ skip,
                             int32_t n_groups, int64_t out_cap, const SnapMeta* __restrict__ meta,
                             GroupMin* __restrict__ gmins, PrepApp* __restrict__ prep, int* __restrict__ err,
                             volatile int* __restrict__ err_host);

// device views of one batch
struct DevApps {
    AppColumns cols;                 // device pointers; cols.off may be NULL (derived on the device)
    const uint8_t* skip;
    int32_t n;
};
struct DevResults {
    int32_t* driver;
    void* exec;                      // int32 or uint16
    int64_t cap;
    int node_bits;
};

gp_status pack_begin(gp_ctx* c, int32_t q, gp_algo algo, gp_mode mode, int64_t exec_cap, bool derive_off, int2** scratch, cudaStream_t st,
                     bool status_in_kernel = false);
gp_status pack_device_range(gp_ctx* c, const DevApps& da, int32_t lo, int32_t hi, int64_t off_base, gp_algo algo, gp_mode mode,
                            const DevResults& dr, int2* scratch, cudaStream_t st, int chunk, bool status_in_kernel = false,
                            bool after_layout = false);
gp_status host_error(gp_ctx* c);

// ---- gangpack_overhead_table.cu --------------------------------------------------------------------------------------

// Enqueue GetOverhead and GetNonSchedulableOverhead of the live overhead table into out[6][n_rows] (overhead cpu, mem, gpu,
// then non-schedulable), a slot counting towards row_of_node[its node id] (-1: none).  Scratch is the caller's: acc
// [12 * n_rows] and *n_warned zeroed, has_reservation [n_slots] or NULL.  *d_err receives the query's bits, decoded by
// oht_sum_refusal once the stream has been synchronised.
void oht_enqueue_sums(gp_ctx* c, cudaStream_t st, const int32_t* row_of_node, int32_t n_rows, unsigned long long* acc,
                      unsigned long long* n_warned, long long* out, uint8_t* has_reservation, int* d_err);
gp_status oht_sum_refusal(gp_ctx* c, int word, const char* who);

// ---- gangpack_cluster.cu ---------------------------------------------------------------------------------------------

// Enqueue gp_resident_dirs over one id array: dir[ids[i]] = i for every ids[i] != -1 (dir [lim] memset to -1 by the caller);
// an id out of [0, lim) or given twice sets *d_err nonzero.  The marker's overhead-table directory.
void enqueue_resident_dir(cudaStream_t st, int32_t n, const int32_t* ids, int32_t lim, int32_t* dir, int* d_err);

// ---- gangpack_reservation_table.cu -----------------------------------------------------------------------------------

// The live reservation table's columns on the device: node id [n_slots] (-1 = free) and cpu / mem / gpu [n_slots] each
struct RtCols { const int32_t* node; const long long* v[3]; };
RtCols rt_cols(gp_ctx* c);

// ---- gangpack_label_table.cu -----------------------------------------------------------------------------------------

// The live label table's columns on the device: count [n_node_ids], key / val [n_node_ids * max_labels], val_int / val_int_ok
// [n_values]
struct LtCols { const int32_t* count; const int32_t* key; const int32_t* val; const long long* vint; const uint8_t* vok; };
LtCols lt_cols(gp_ctx* c);

// ---- gangpack_node_table.cu ------------------------------------------------------------------------------------------

// What a *_node_table entry hands to the *_resident stages: a gp_resident_usage and a gp_sort_input over the listed nodes whose
// columns (is_driver_candidate and the id arrays excepted) are device pointers into the context's gather buffer, the
// instance groups (device, or NULL), and the gather's status word, read by the stage's one synchronise (nt_refusal).
struct NtGathered {
    gp_resident_usage usage;
    gp_sort_input sort;
    const int32_t* ig;
    const long long* creation;                // the failover reconciler's creation times (NtReconcile given), else NULL
    const int* err;
};
// The failover reconciler's instance groups: instanceGroup(n.Labels[key]) in [0, n_groups), a missing label in `missing`
// (the dense id of "", -1 refused), a value not listed refused; key -1: every node in 0.  The gather then writes creation too.
struct NtReconcile {
    int32_t missing;
};
// The host checks of a *_node_table entry, then the gather enqueued on the context's stream.  ig_host (or NULL): the entry's
// instance_group array, uploaded as is (checked by the *_resident entry); with_ig: read instance groups from the labels.
// recon: the reconciler's rule over n_ig groups instead of the Predicates' (with_ig true, ig_host NULL).  reservations false:
// reservation_id may be NULL (the marker's entries).
gp_status nt_gather(gp_ctx* c, const gp_node_table_nodes* nodes, const int32_t* ig_host, int32_t n_ig, bool with_ig, const char* who,
                    NtGathered* out, const NtReconcile* recon = nullptr, bool reservations = true);
// The gather's refusal, once the stream has been synchronised
gp_status nt_refusal(gp_ctx* c, int word, const char* who);
// After the entry's synchronise: the optional zone_id_out / instance_group_out copies
gp_status nt_outputs(gp_ctx* c, const gp_node_table_nodes* nodes, const NtGathered& g);

// ---- gangpack_driver_table.cu ----------------------------------------------------------------------------------------

// The stale drivers of one marker sweep as device columns in (creation, slot) order, in the driver table's queue buffer: the
// six quantities, count and capacity group (the affinity id, -1 -> n_aff) of each, all zero for a row outside the model
struct DtStale {
    int32_t n;
    const int64_t* q[6];
    const int32_t* count;
    const int32_t* group;
};
// The stale stage of gp_exceeds_cluster_capacity_driver_table over a live driver table: select, order and scatter, one
// synchronise, then the refusals (an affinity id outside [-1, n_aff) on a stale row, then n_stale > cap with *n_stale
// written).  stale_slot and outcome (0, or 2 outside the model) are downloaded on the stream: complete after the next
// synchronise.
gp_status dt_stale_stage(gp_ctx* c, const gp_stale_sweep* sw, int32_t n_aff, const char* who, DtStale* out);

// ---- gangpack_zones.cu -----------------------------------------------------------------------------------------------

// The applications of one zone FIFO drain: host columns to upload (host, with group = their instance groups or NULL and off
// = the offsets), or (host NULL) device columns already in instance-group order, queue order within each: q[6] the six
// quantities (NULL = 0), count, off, skip and queue = the identity over the applications.
struct ZoneFifoApps {
    const gp_apps* host;
    const int32_t* group;
    const int64_t* off;
    const int64_t* q[6];
    const int32_t* count;
    const uint8_t* skip;
    const int32_t* queue;
};
// gp_pack_fifo_zones_groups' packer and mode checks: kind = GP_TIGHTLY_PACK / GP_MINIMAL_FRAGMENTATION / kZoneAzAware
gp_status zone_fifo_kind(gp_ctx* c, gp_binpacker packer, gp_mode mode, const char* who, int* kind);
// The layout gp_prepare_cluster_zones_groups left (groups == NULL), checked for the packer kind
gp_status held_groups_layout(gp_ctx* c, int kind, const char* who, gp_instance_groups* held);
// The zone FIFO drain over Q applications with `total` ExecutorNodes entries; c->zone_groups [n_instance_groups] holds each
// instance group's application count in q_end and its largest exe_count in row_pitch
gp_status fifo_zones_body(gp_ctx* c, int32_t Q, int64_t total, const ZoneFifoApps& src, int kind, gp_mode mode,
                          const gp_instance_groups& ig, bool az_dev, gp_zone_results* out, const char* who);

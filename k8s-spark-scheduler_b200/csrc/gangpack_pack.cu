// gangpack_pack.cu -- gp_pack_batch and its variants (gp_pack_batch_wire, gp_pack_batch_device, gp_pack_one) and
// gp_last_stats: the independent and FIFO pack launches, the pipelined batch path, and the pack steps the zone entry
// points reuse (pack_begin, pack_device_range, host_error).
#include "gangpack_ctx.cuh"
#include "gangpack_fifo.cuh"
#include "gangpack_minfrag.cuh"
#include "gangpack_tables.cuh"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <string>

// Thread per application: validate, derive the division magics and the driver-displacement bound (FIFO modes and
// minimal-fragmentation; independent tightly-pack / distribute-evenly prepare inside gp_pack_tables).
// Source tuple: types.SparkApplicationResources (internal/types/types.go:22-27).
__global__ void gp_prep_apps(int32_t n_apps, AppColumns cols, const uint8_t* __restrict__ skip,
                             int32_t n_groups, int64_t out_cap, const SnapMeta* __restrict__ meta,
                             GroupMin* __restrict__ gmins, PrepApp* __restrict__ prep, int* __restrict__ err,
                             volatile int* __restrict__ err_host) {
    // records are staged in shared memory and written out with fully coalesced 16-byte stores (a thread writing
    // its own 128-byte record would touch 32 different lines per warp-wide store)
    __shared__ uint4 stage[kPrepThreads * (sizeof(PrepApp) / sizeof(uint4))];
    const int32_t block0 = blockIdx.x * blockDim.x;
    int32_t i = block0 + threadIdx.x;
    const bool live = i < n_apps;
    if (!live) i = n_apps - 1;                      // keep the thread for the cooperative copy-out; its record is not stored
    int64_t d[3] = {cols.load(0, i), cols.load(1, i), cols.load(2, i)};
    int64_t e[3] = {cols.load(3, i), cols.load(4, i), cols.load(5, i)};
    int32_t k = cols.count[i];
    int32_t g = cols.group ? cols.group[i] : 0;
    int bad = 0;
    if (k < 0) bad |= kErrNegativeRequest;
    if (k > kMaxCount) bad |= kErrUnrepresentable;
    if (gmins && k > kMaxCountFifo) bad |= kErrUnrepresentable;   // FIFO modes: block-wide uint32 sums of clamped capacities stay exact
    if (g < 0 || g >= n_groups) bad |= kErrBadGroup;
    int64_t off = cols.off[i];
    if (off < 0 || cols.off[i + 1] - off != (int64_t)k || cols.off[i + 1] > out_cap) bad |= kErrBadOffsets;
    PrepApp p;
    uint64_t lmax = 0;
    bool fast = true;
#pragma unroll
    for (int t = 0; t < 3; ++t) {
        uint64_t l;
        p.drv[t] = d[t];
        p.div[t] = prep_dim(d[t], e[t], t, meta->max_avail[t], bad, l, fast);
        if (l > lmax) lmax = l;
    }
    if (bad && live) { atomicOr(err, bad); *err_host = bad; }   // err_host: mapped pinned word, no D2H copy needed
    if (bad) { k = 0; g = 0; }
    else if (gmins && live) {
        // batch-wide minima per instance group (FIFO dead-node skipping)
        GroupMin* gm = gmins + g;
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            if (e[t] < gm->exe[t]) atomicMin(&gm->exe[t], (long long)e[t]);
            if (d[t] < gm->drv[t]) atomicMin(&gm->drv[t], (long long)d[t]);
        }
    }
    p.out_off = off;
    p.count = k;
    p.group = g;
    p.lmax = (int32_t)(lmax < (uint64_t)k ? lmax : (uint64_t)k);
    const bool fast32 = prep_fast32(fast, p.div[0], p.div[1], meta);
    p.flags = ((d[2] != 0 || e[2] != 0) ? kAppUsesGpu : 0u) | ((skip && skip[i]) ? kAppSkipIfNoFit : 0u) |
              (bad ? kAppInvalid : 0u) | (fast ? kAppFast : 0u) | (fast32 ? kAppFast32 : 0u);
    constexpr int kQ = sizeof(PrepApp) / sizeof(uint4);      // 8 x 16 bytes per record
    const uint4* src = reinterpret_cast<const uint4*>(&p);
#pragma unroll
    for (int w = 0; w < kQ; ++w) stage[threadIdx.x * kQ + w] = src[w];
    __syncthreads();
    const int32_t n_block = min((int32_t)blockDim.x, n_apps - block0);
    uint4* dst = reinterpret_cast<uint4*>(prep + block0);
    for (int32_t t = threadIdx.x; t < n_block * kQ; t += blockDim.x) dst[t] = stage[t];
}

// Independent minimal-fragmentation (GP_MODE_INDEPENDENT): one warp per application; warps claim applications from a
// global counter (claim-then-broadcast, next index prefetched) so long scans do not leave a tail.  Independent
// tightly-pack / distribute-evenly take gp_decide_tables instead.
constexpr int kPackThreads = 256;
template <int ALGO>
#ifndef GP_MF_MIN_BLOCKS
#define GP_MF_MIN_BLOCKS 4      // minimal-fragmentation: 64 registers (96 uncapped); occupancy hides its dependent multi-pass loads
#endif
__global__ void __launch_bounds__(kPackThreads, GP_MF_MIN_BLOCKS) gp_pack_independent(Snapshot s, const PrepApp* __restrict__ prep, int32_t n_apps,
                                                                    int32_t* __restrict__ driver_node,
                                                                    int32_t* __restrict__ executor_nodes,
                                                                    int2* __restrict__ scratch,
                                                                    unsigned long long* __restrict__ stats,
                                                                    unsigned int* __restrict__ next_app) {
    static_assert(ALGO == 2, "gp_pack_independent is minimal-fragmentation only");
    const int lane = threadIdx.x & 31;
    WarpStats st{0, 0};
    const int snap_flags = s.meta->flags;          // per-kernel facts stay in registers
    // claim-then-broadcast, two applications ahead: while application i is packed, the index of i+2 is in
    // flight and the record of i+1 is being pulled into L1
    unsigned int i = 0, n1 = 0;
    if (lane == 0) { i = atomicAdd(next_app, 1u); n1 = atomicAdd(next_app, 1u); }
    i = __shfl_sync(kFull, i, 0);
    n1 = __shfl_sync(kFull, n1, 0);
    while (i < (unsigned int)n_apps) {
        unsigned int n2 = 0;
        if (lane == 0) n2 = atomicAdd(next_app, 1u);
        if (lane == 0 && n1 < (unsigned int)n_apps) asm volatile("prefetch.global.L1 [%0];" ::"l"(prep + n1));
        const PrepApp* pa = prep + i;
        int32_t d = -1;
        if (!(pa->flags & kAppInvalid)) {       // multi-pass, see gangpack_minfrag.cuh
            const bool gpu_idle = !(pa->flags & kAppUsesGpu) && !(snap_flags & kSnapGpuNegative);
            d = ((pa->flags & kAppFast32) && gpu_idle) ? pack_app_minfrag<true>(s, pa, executor_nodes, scratch, st, lane, snap_flags)
                                                       : pack_app_minfrag<false>(s, pa, executor_nodes, scratch, st, lane, snap_flags);
        }
        if (lane == 0) driver_node[i] = d;
        i = n1;
        n1 = __shfl_sync(kFull, n2, 0);
    }
    if (lane == 0) {
        atomicAdd(stats + 0, st.nodes);
        atomicAdd(stats + 1, st.drivers);
    }
}

// ---- packing ------------------------------------------------------------------------------------

static AppColumns cols_at(const AppColumns& c, int32_t lo) {
    AppColumns r = c;
    const size_t es = c.bits == 64 ? 8 : 4;
    for (int k = 0; k < 6; ++k) if (c.q[k]) r.q[k] = static_cast<const char*>(c.q[k]) + es * (size_t)lo;
    r.count = c.count + lo;
    if (c.group) r.group = c.group + lo;
    if (c.off) r.off = c.off + lo;
    return r;
}

// independent minimal-fragmentation: persistent grid, as many CTAs as fit on the device (or fewer for small batches)
static void launch_minfrag(gp_ctx* c, const Snapshot& s, const PrepApp* prep, int32_t n_apps, int32_t* driver_node,
                           int32_t* executor_nodes, int2* scratch, unsigned long long* stats, unsigned int* next_app, cudaStream_t st) {
    int& per_sm = c->pack_ctas_per_sm;
    if (per_sm == 0) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gp_pack_independent<2>, kPackThreads, 0);
        if (per_sm < 1) per_sm = 1;
    }
    int64_t blocks = ((int64_t)n_apps * 32 + kPackThreads - 1) / kPackThreads;
    int64_t max_blocks = (int64_t)c->sm_count * per_sm;
    if (blocks > max_blocks) blocks = max_blocks;
    if (blocks < 1) blocks = 1;
    gp_pack_independent<2><<<(int)blocks, kPackThreads, 0, st>>>(s, prep, n_apps, driver_node, executor_nodes, scratch, stats, next_app);
}

// FIFO modes (tightly-pack / distribute-evenly): one persistent 1024-thread CTA per instance group, its slots staged in
// shared memory
template <int ALGO>
static gp_status launch_fifo(gp_ctx* c, gp_mode mode, const Snapshot& s, const PrepApp* prep, const int32_t* app_group, int32_t n_apps,
                             int32_t* driver_node, int32_t* executor_nodes, int2* scratch, unsigned long long* stats, cudaStream_t st) {
    const auto kernels = {gp_pack_fifo_cta<ALGO, 1, true>, gp_pack_fifo_cta<ALGO, 2, true>, gp_pack_fifo_cta<ALGO, 1, false>,
                          gp_pack_fifo_cta<ALGO, 2, false>};
    bool& attr_set = c->fifo_attr_set[ALGO];     // per device: function attributes live in the device's context
    if (!attr_set) {
        for (auto k : kernels) GP_CUDA(c, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFifoSmemBytes));
        attr_set = true;
    }
    auto kern = mode == GP_MODE_FIFO_REFERENCE ? (c->fifo_warp ? gp_pack_fifo_cta<ALGO, 1, true> : gp_pack_fifo_cta<ALGO, 1, false>)
                                               : (c->fifo_warp ? gp_pack_fifo_cta<ALGO, 2, true> : gp_pack_fifo_cta<ALGO, 2, false>);
    kern<<<s.n_groups, kFifoThreads, kFifoSmemBytes, st>>>(s, prep, app_group, n_apps, driver_node, executor_nodes, scratch, stats, s.gmins,
                                                           c->fifo_list.as<int32_t>(), &c->status()->fifo_cursor);
    // the FIFO kernels subtract usage from `pair` in place: refresh the compact 32-bit view so that a later
    // independent pack on this context (the driver's own pack after fitEarlierDrivers, resource.go:255 then :321)
    // sees the charged availability
    const int T = 256;
    gp_fill_pair32<<<(c->n_slots + T) / T, T, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), c->snap_flags.as<SnapMeta>(), c->pair32.as<uint2>());
    c->last.kernel_launches += 1;
    return GP_OK;
}

// independent tightly-pack / distribute-evenly: one launch for classify -> capacity tables -> thread-per-application
// decisions, then the warp-per-application scan of whatever the tables could not decide (gangpack_tables.cuh)
template <int ALGO, class OUT>
static gp_status launch_tables(gp_ctx* c, const Snapshot& s, const AppColumns& cols, const ShapeTables& tabs, int64_t off_base,
                               int64_t* off_out, int32_t* app_slot, PrepApp* prep, int32_t* listed, int32_t q, const DevResults& dr,
                               int32_t lo, int2* scratch, unsigned long long* stats, unsigned int* next_app, int* d_err,
                               volatile int* err_host, bool use_tables, int64_t seg_bound, unsigned int* status_zero, bool early_start,
                               cudaStream_t st) {
    int& dec_per_sm = c->dec_ctas_per_sm[ALGO][sizeof(OUT) == 2 ? 1 : 0];
    if (dec_per_sm == 0) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&dec_per_sm, gp_decide_tables<ALGO, OUT>, kTabThreads, 0);
        if (dec_per_sm < 1) dec_per_sm = 1;
    }
    // persistent grid: as many CTAs as fit on the device, or as many as there can be work items
    const int64_t tiles = ((int64_t)q + kTabThreads - 1) / kTabThreads;
    const int64_t shapes = std::min<int64_t>(q, kMaxShapes);
    int64_t blocks = tiles * ((use_tables || off_out) ? 2 : 1) + (use_tables ? shapes * (seg_bound + c->n_groups) : 0);
    blocks = std::min<int64_t>(blocks, (int64_t)c->sm_count * dec_per_sm);
    // early_start: it may start while the slot layout before it on st still runs (see gp_decide_tables)
    GP_CUDA(c, launch_pdl(early_start, (int)blocks, kTabThreads, st, gp_decide_tables<ALGO, OUT>, s, cols, tabs, off_base, off_out, app_slot,
                          q, dr.cap, dr.driver + lo, static_cast<OUT*>(dr.exec), prep, listed, stats, d_err, err_host,
                          use_tables ? 0 : 1, status_zero));
    int& per_sm = c->tab_ctas_per_sm[ALGO][sizeof(OUT) == 2 ? 1 : 0];
    if (per_sm == 0) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gp_pack_listed<ALGO, OUT>, kPackTabThreads, 0);
        if (per_sm < 1) per_sm = 1;
    }
    // persistent grid; with the tables on the list is normally short (or empty: the CTAs leave at once)
    blocks = ((int64_t)q * 32 + kPackTabThreads - 1) / kPackTabThreads;
    const int64_t max_blocks = (int64_t)c->sm_count * (use_tables ? 2 : per_sm);
    if (blocks > max_blocks) blocks = max_blocks;
    if (blocks < 1) blocks = 1;
    // it also zeroes the classify tiles' and the table segments' look-back words (see there); it waits for
    // gp_decide_tables before it reads or writes anything
    GP_CUDA(c, launch_pdl(true, (int)blocks, kPackTabThreads, st, gp_pack_listed<ALGO, OUT>, s, tabs, (int32_t)tiles,
                          use_tables ? kMaxShapes * (int32_t)seg_bound : 0, prep, listed, dr.driver + lo, static_cast<OUT*>(dr.exec),
                          scratch, stats, next_app));
    c->last.kernel_launches += 2;
    return GP_OK;
}

// Device-resident apps [lo, hi): enqueue the kernels on `st`; chunk index selects the timing events and the table lane.
// off_base: ExecutorNodes offset of application `lo` (only used when the offsets are derived on the device).
// status_in_kernel: pack_begin left the status block to this range's decide kernel (kernel_zeroes_status(), one range only).
// after_layout: the last work on st is this context's slot layout, and the caller's inputs were ready before it was
// enqueued (Held::take_tail).
gp_status pack_device_range(gp_ctx* c, const DevApps& da, int32_t lo, int32_t hi, int64_t off_base, gp_algo algo, gp_mode mode,
                            const DevResults& dr, int2* scratch, cudaStream_t st, int chunk, bool status_in_kernel, bool after_layout) {
    const int32_t q = hi - lo;
    if (q <= 0) return GP_OK;
    int* d_err = &c->status()->head.err;
    unsigned long long* d_stats = c->status()->head.stats;
    unsigned int* next_app = &c->status()->next_app[chunk];
    volatile int* err_host = &c->host_status()->err_word;
    Snapshot s = make_snapshot(c);
    AppColumns cols = cols_at(da.cols, lo);

    if (mode == GP_MODE_INDEPENDENT && algo != GP_MINIMAL_FRAGMENTATION) {
        gp_ctx::TableSet& T = c->tabs[chunk % gp_ctx::kLanes];
        const bool use_tables = c->use_tables && q >= 32;
        int64_t* off_out = nullptr;
        if (!da.cols.off) {                       // derive the offsets on the device
            off_out = c->off_dev.as<int64_t>() + lo;
            cols.off = off_out;
        }
        // [header | executor hash | driver hash | look-back words of the classify tiles | look-back words of the table
        // segments]: zeroed when allocated, and gp_pack_listed zeroes what each call used of it.  The hash entries sit at
        // the same place whatever q is, so the words a later call expects zero never overlap the fields a claimer wrote.
        const size_t n_tiles = ((size_t)q + kTabThreads - 1) / kTabThreads;
        const size_t cls_bytes = (sizeof(unsigned long long) * n_tiles + 15) & ~(size_t)15;
        const size_t hash_bytes = (sizeof(ShapeEntry) + sizeof(DriverEntry)) * (size_t)kShapeSlots;
        // sum over the groups of max(1, ceil(ne / kTabSeg)) <= n_slots / kTabSeg + n_groups
        const int64_t seg_bound = (int64_t)c->n_slots / kTabSeg + c->n_groups + 1;
        const size_t hdr_bytes = 1024 + hash_bytes + cls_bytes + sizeof(unsigned long long) * (size_t)kMaxShapes * (size_t)seg_bound;
        const size_t hdr_cap = T.hdr.cap;
        GP_CUDA(c, T.hdr.reserve_zeroed(hdr_bytes, st));
        // gp_decide_tables may start before the layout ends only when it is the first work this call enqueues: neither
        // pack_begin's status memset nor the header's zeroing above (a timing event is no work)
        const bool early_start = after_layout && status_in_kernel && T.hdr.cap == hdr_cap;
        // [executor slot | driver slot | listed]
        GP_CUDA(c, T.app_slot.reserve(sizeof(int32_t) * (3 * (size_t)q + 1)));
        if (use_tables) {
            GP_CUDA(c, T.table.reserve(sizeof(uint32_t) * (size_t)kMaxShapes * (size_t)((c->n_slots + 4) & ~3)));
            // total | firstfit | first_host
            GP_CUDA(c, T.total.reserve(sizeof(uint32_t) * 3 * (size_t)kMaxShapes * (size_t)c->n_groups));
            GP_CUDA(c, T.place.reserve(sizeof(int32_t) * (size_t)kMaxShapes * (size_t)c->n_groups * kPlaceLen));
        }
        ShapeTables tabs;
        tabs.hdr = T.hdr.as<ShapeHeader>();
        tabs.entries = reinterpret_cast<ShapeEntry*>(T.hdr.as<char>() + 1024);
        tabs.dentries = reinterpret_cast<DriverEntry*>(T.hdr.as<char>() + 1024 + sizeof(ShapeEntry) * (size_t)kShapeSlots);
        tabs.cls_status = reinterpret_cast<unsigned long long*>(T.hdr.as<char>() + 1024 + hash_bytes);
        tabs.seg_status = reinterpret_cast<unsigned long long*>(T.hdr.as<char>() + 1024 + hash_bytes + cls_bytes);
        tabs.table = T.table.as<uint32_t>(); tabs.total = T.total.as<uint32_t>();
        tabs.firstfit = reinterpret_cast<int32_t*>(T.total.as<uint32_t>() + (size_t)kMaxShapes * (size_t)c->n_groups);
        tabs.first_host = tabs.firstfit + (size_t)kMaxShapes * (size_t)c->n_groups;
        tabs.seg_pre = c->seg_pre.as<int32_t>();
        tabs.place = T.place.as<int32_t>();
        tabs.pitch = (c->n_slots + 4) & ~3; tabs.n_groups = c->n_groups;      // rows start 16-byte aligned
        int32_t* app_slot = T.app_slot.as<int32_t>();
        int32_t* listed = app_slot + 2 * (size_t)q;
        PrepApp* prep = c->prep.as<PrepApp>() + lo;
        const bool o16 = dr.node_bits == 16;
        const auto launch = algo == GP_TIGHTLY_PACK ? (o16 ? launch_tables<0, uint16_t> : launch_tables<0, int32_t>)
                                                    : (o16 ? launch_tables<1, uint16_t> : launch_tables<1, int32_t>);
        unsigned int* status_zero = status_in_kernel ? reinterpret_cast<unsigned int*>(c->status()) : nullptr;
        c->ev_prep = false;                            // one launch prepares and packs: no separate prep interval
        auto issue = [&](int& launches) -> gp_status {
            const int before = (int)c->last.kernel_launches;
            if (c->record_events) GP_CUDA(c, cudaEventRecord(c->ev[chunk][1], st));
            const gp_status r = launch(c, s, cols, tabs, off_base, off_out, app_slot, prep, listed, q, dr, lo, scratch, d_stats, next_app,
                                       d_err, err_host, use_tables, seg_bound, status_zero, early_start, st);
            if (r != GP_OK) return r;
            GP_CUDA(c, cudaGetLastError());
            if (c->record_events) GP_CUDA(c, cudaEventRecord(c->ev[chunk][2], st));
            launches = (int)c->last.kernel_launches - before;
            c->last.kernel_launches = before;          // run_cached adds `launches` (also when the graph is replayed)
            return GP_OK;
        };
        if (c->record_events) {                        // timing events inside: always issued directly
            int n = 0;
            gp_status r = issue(n);
            c->last.kernel_launches += n;
            return r;
        }
        struct { int32_t algo, o16, use_tables, q, lo, chunk, early_start; int64_t off_base; AppColumns cols; ShapeTables tabs; Snapshot snap;
                 const void* p[11]; int64_t cap; } key{};
        key.algo = (int32_t)algo; key.o16 = o16; key.use_tables = use_tables; key.q = q; key.lo = lo; key.chunk = chunk; key.early_start = early_start; key.off_base = off_base;
        key.cols = cols; key.tabs = tabs; key.snap = s; key.cap = dr.cap;
        const void* ptrs[11] = {app_slot, prep, listed, dr.driver, dr.exec, scratch, d_stats, next_app, d_err, off_out, status_zero};
        std::memcpy(key.p, ptrs, sizeof(ptrs));
        return run_cached(c, c->g_chunk[st == c->stream ? kMaxChunks : chunk], &key, sizeof(key), st, issue);
    }

    // ---- FIFO modes and minimal-fragmentation: prepared records + the pack kernel ------------------------------------
    PrepApp* prep = c->prep.as<PrepApp>() + lo;
    const int T = kPrepThreads;
    if (mode != GP_MODE_INDEPENDENT) {
        GP_CUDA(c, c->fifo_list.reserve(sizeof(int32_t) * (size_t)(q + 1)));
        GP_CUDA(c, c->gmin.reserve(sizeof(GroupMin) * (size_t)c->n_groups));
        GP_CUDA(c, cudaMemsetAsync(c->gmin.p, 0x7f, sizeof(GroupMin) * (size_t)c->n_groups, st));   // +inf-ish
    }
    c->ev_prep = true;
    if (c->record_events) GP_CUDA(c, cudaEventRecord(c->ev[chunk][0], st));
    gp_prep_apps<<<(q + T - 1) / T, T, 0, st>>>(
        q, cols, da.skip ? da.skip + lo : nullptr, c->n_groups, dr.cap,
        c->snap_flags.as<SnapMeta>(), mode == GP_MODE_INDEPENDENT ? nullptr : c->gmin.as<GroupMin>(), prep, d_err, err_host);
    s.gmins = c->gmin.as<GroupMin>();
    if (c->record_events) GP_CUDA(c, cudaEventRecord(c->ev[chunk][1], st));
    int32_t* exec32 = static_cast<int32_t*>(dr.exec);
    if (mode == GP_MODE_INDEPENDENT) {
        launch_minfrag(c, s, prep, q, dr.driver + lo, exec32, scratch, d_stats, next_app, st);
    } else {                              // (check_args rejects the FIFO modes for minimal-fragmentation)
        const gp_status r = algo == GP_TIGHTLY_PACK ? launch_fifo<0>(c, mode, s, prep, cols.group, q, dr.driver + lo, exec32, scratch, d_stats, st)
                                                    : launch_fifo<1>(c, mode, s, prep, cols.group, q, dr.driver + lo, exec32, scratch, d_stats, st);
        if (r != GP_OK) return r;
    }
    GP_CUDA(c, cudaGetLastError());
    if (c->record_events) GP_CUDA(c, cudaEventRecord(c->ev[chunk][2], st));
    c->last.kernel_launches += 2;
    return GP_OK;
}

static bool fused_path(gp_algo algo, gp_mode mode) { return mode == GP_MODE_INDEPENDENT && algo != GP_MINIMAL_FRAGMENTATION; }

// One range of q > 0 independent tightly-pack / distribute-evenly applications on one stream: the first classify tile of
// its decide kernel zeroes the status block (gp_decide_tables), so pack_begin leaves out its memset.  Calls that pack
// several ranges or take other kernels keep the memset.
static bool kernel_zeroes_status(int32_t q, gp_algo algo, gp_mode mode) { return q > 0 && fused_path(algo, mode); }

// common prologue: buffers, counters
gp_status pack_begin(gp_ctx* c, int32_t q, gp_algo algo, gp_mode mode, int64_t exec_cap, bool derive_off, int2** scratch, cudaStream_t st,
                     bool status_in_kernel) {
    if (!status_in_kernel) GP_CUDA(c, cudaMemsetAsync(c->status(), 0, sizeof(DevStatus), st));
    c->host_status()->err_word = 0;
    c->last = gp_stats{};
    c->ev_chunks = 0;
    *scratch = nullptr;
    if (q == 0) return GP_OK;
    GP_CUDA(c, c->prep.reserve(sizeof(PrepApp) * (size_t)q));      // FIFO / minimal-fragmentation: every application; tables: the listed ones
    if (derive_off) GP_CUDA(c, c->off_dev.reserve(sizeof(int64_t) * (size_t)(q + 1)));
    if (algo != GP_TIGHTLY_PACK) {        // candidate list (distribute-evenly) / consumed-node list (minimal-fragmentation)
        GP_CUDA(c, c->scratch.reserve(sizeof(int2) * (size_t)(exec_cap + 1)));
        *scratch = c->scratch.as<int2>();
    }
    return GP_OK;
}

static gp_status check_args(gp_ctx* c, const gp_apps_wire* a, gp_algo algo, gp_mode mode, const gp_results_wire* out, const char* who) {
    GP_TRY(require(c, c->held.snapshot(), who));
    if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, std::string(who) + ": NULL apps/results");
    if (algo != GP_TIGHTLY_PACK && algo != GP_DISTRIBUTE_EVENLY && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, std::string(who) + ": unknown algo");
    if (algo == GP_MINIMAL_FRAGMENTATION && mode != GP_MODE_INDEPENDENT)
        return fail(c, GP_ERR_INVALID, std::string(who) + ": minimal-fragmentation is offered in GP_MODE_INDEPENDENT only "
                                                          "(its one registered caller, single-az-minimal-fragmentation, chooses a zone per application on the host)");
    if (mode != GP_MODE_INDEPENDENT && mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, std::string(who) + ": unknown mode");
    if (a->quantity_bits != 64 && a->quantity_bits != 32) return fail(c, GP_ERR_INVALID, std::string(who) + ": quantity_bits must be 64 or 32");
    if (a->quantity_bits == 32 && (a->mem_shift < 0 || a->mem_shift > 40)) return fail(c, GP_ERR_INVALID, std::string(who) + ": mem_shift out of range");
    if (out->node_bits != 32 && out->node_bits != 16) return fail(c, GP_ERR_INVALID, std::string(who) + ": node_bits must be 32 or 16");
    if (out->node_bits == 16 && (!fused_path(algo, mode) || c->n_nodes > 65535))
        return fail(c, GP_ERR_INVALID, std::string(who) + ": 16-bit node indices need <= 65535 nodes and GP_MODE_INDEPENDENT tightly-pack / distribute-evenly");
    if (a->n_apps > 0 && (!a->drv_cpu || !a->drv_mem || !a->exe_cpu || !a->exe_mem || !a->exe_count || !out->driver_node))
        return fail(c, GP_ERR_INVALID, std::string(who) + ": missing app/result arrays");
    if (a->n_apps > 0 && !a->exec_out_off && !fused_path(algo, mode))
        return fail(c, GP_ERR_INVALID, std::string(who) + ": exec_out_off may only be NULL for GP_MODE_INDEPENDENT tightly-pack / distribute-evenly");
    return GP_OK;
}

// after the streams have been synchronised: event times of the last pack, summed over its chunks
static void fill_kernel_times(gp_ctx* c) {
    c->last.prep_kernel_ns = 0; c->last.pack_kernel_ns = 0;
    for (int i = 0; i < c->ev_chunks; ++i) {
        float a = 0.f, b = 0.f;
        if (c->ev_prep && cudaEventElapsedTime(&a, c->ev[i][0], c->ev[i][1]) == cudaSuccess) c->last.prep_kernel_ns += (int64_t)(a * 1.0e6);
        if (cudaEventElapsedTime(&b, c->ev[i][1], c->ev[i][2]) == cudaSuccess) c->last.pack_kernel_ns += (int64_t)(b * 1.0e6);
    }
}

static gp_status decode_device_error(gp_ctx* c, int err) {
    if (err == 0) return GP_OK;
    if (err & kErrUnrepresentable) return fail(c, GP_ERR_UNREPRESENTABLE, "pack: quantity >= 2^61 or exe_count > 2^24 (2^20 in the FIFO modes)");
    if (err & kErrNegativeRequest) return fail(c, GP_ERR_INVALID, "pack: negative resource request or executor count");
    if (err & kErrBadGroup) return fail(c, GP_ERR_INVALID, "pack: app group out of range");
    return fail(c, GP_ERR_CAPACITY, "pack: exec_out_off inconsistent with exe_count or executor_nodes_cap too small");
}

// after a synchronise: the validation errors the kernels reported through the mapped error word
gp_status host_error(gp_ctx* c) { return decode_device_error(c, c->host_status()->err_word); }

static gp_apps_wire widen(const gp_apps* a) {
    gp_apps_wire w{};
    w.n_apps = a->n_apps; w.quantity_bits = 64; w.mem_shift = 0;
    w.drv_cpu = a->drv_cpu_milli; w.drv_mem = a->drv_mem_bytes; w.drv_gpu = a->drv_gpu;
    w.exe_cpu = a->exe_cpu_milli; w.exe_mem = a->exe_mem_bytes; w.exe_gpu = a->exe_gpu;
    w.exe_count = a->exe_count; w.group = a->group; w.skip_if_no_fit = a->skip_if_no_fit; w.exec_out_off = a->exec_out_off;
    return w;
}

extern "C" {

gp_status gp_pack_batch_device(gp_ctx* c, const gp_apps* da, gp_algo algo, gp_mode mode, gp_results* dout, void* stream) {
    const void* layout_tail = nullptr;
    if (!enter(c, &layout_tail)) return GP_ERR_INVALID;
    if (!da || !dout) return fail(c, GP_ERR_INVALID, "gp_pack_batch_device: NULL apps/results");
    const gp_apps_wire w = widen(da);
    gp_results_wire ow{dout->driver_node, dout->executor_nodes, dout->executor_nodes_cap, 32, 0};
    gp_status s = check_args(c, &w, algo, mode, &ow, "gp_pack_batch_device");
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream;
    int2* scratch = nullptr;
    const bool zero_in_kernel = kernel_zeroes_status(w.n_apps, algo, mode);
    const bool after_layout = layout_tail == st;
    s = pack_begin(c, w.n_apps, algo, mode, ow.executor_nodes_cap, !w.exec_out_off, &scratch, st, zero_in_kernel);
    if (s != GP_OK || w.n_apps == 0) return s;
    DevApps dv{};
    dv.cols.q[0] = w.drv_cpu; dv.cols.q[1] = w.drv_mem; dv.cols.q[2] = w.drv_gpu;
    dv.cols.q[3] = w.exe_cpu; dv.cols.q[4] = w.exe_mem; dv.cols.q[5] = w.exe_gpu;
    dv.cols.count = w.exe_count; dv.cols.group = w.group; dv.cols.off = w.exec_out_off; dv.cols.bits = 64; dv.cols.mem_shift = 0;
    dv.skip = w.skip_if_no_fit; dv.n = w.n_apps;
    DevResults dr{ow.driver_node, ow.executor_nodes, ow.executor_nodes_cap, 32};
    s = pack_device_range(c, dv, 0, w.n_apps, 0, algo, mode, dr, scratch, st, 0, zero_in_kernel, after_layout);
    if (s == GP_OK) c->ev_chunks = 1;
    return s;
}

gp_status gp_last_stats(gp_ctx* c, gp_stats* out) {
    if (!out || !enter(c)) return GP_ERR_INVALID;
    GP_CUDA(c, cudaSetDevice(c->device));
    StatusHead& h = c->host_status()->head;
    GP_CUDA(c, cudaMemcpyAsync(&h, &c->status()->head, sizeof(StatusHead), cudaMemcpyDeviceToHost, c->stream));
    GP_CUDA(c, cudaStreamSynchronize(c->stream));
    c->last.nodes_scanned = (int64_t)h.stats[0];
    c->last.drivers_tried = (int64_t)h.stats[1];
    c->last.scan_path_apps = (int64_t)h.stats[2];
    c->last.scan_path_nodes = (int64_t)h.stats[3];
    fill_kernel_times(c);
    *out = c->last;
    return decode_device_error(c, h.err);
}

#ifdef GP_DECIDE_TIMELINE
// Diagnostic build only (not in gangpack.h): copy the phase timeline of the last gp_decide_tables launch on the context's
// device (gp::TlBuf) into `out`, after the context's stream has finished.  -> the bytes needed; copies only if bytes suffices.
int64_t gp_decide_timeline(gp_ctx* c, void* out, int64_t bytes) {
    if (!c) return -1;
    if (cudaSetDevice(c->device) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) return -1;
    if (out && bytes >= (int64_t)sizeof(gp::TlBuf) && cudaMemcpyFromSymbol(out, gp::g_tl, sizeof(gp::TlBuf)) != cudaSuccess) return -1;
    return (int64_t)sizeof(gp::TlBuf);
}
#endif

static gp_status pack_batch_impl(gp_ctx* c, const gp_apps_wire* a, gp_algo algo, gp_mode mode, gp_results_wire* out);

gp_status gp_pack_batch_wire(gp_ctx* c, const gp_apps_wire* a, gp_algo algo, gp_mode mode, gp_results_wire* out) {
    if (!enter(c)) return GP_ERR_INVALID;
    gp_status s = pack_batch_impl(c, a, algo, mode, out);
    if (s != GP_OK) {
        // Whatever was enqueued before the failure may still read the caller's buffers or write its results:
        // drain every stream of this context before handing control (and buffer ownership) back.
        const std::string keep = c->err;
        cudaSetDevice(c->device);
        for (cudaStream_t l : c->lane) if (l) cudaStreamSynchronize(l);
        if (c->stream) cudaStreamSynchronize(c->stream);
        cudaGetLastError();
        c->err = keep;
    }
    return s;
}

gp_status gp_pack_batch(gp_ctx* c, const gp_apps* a, gp_algo algo, gp_mode mode, gp_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!a || !out) return fail(c, GP_ERR_INVALID, "gp_pack_batch: NULL apps/results");
    const gp_apps_wire w = widen(a);
    gp_results_wire ow{out->driver_node, out->executor_nodes, out->executor_nodes_cap, 32, 0};
    return gp_pack_batch_wire(c, &w, algo, mode, &ow);
}

static gp_status pack_batch_impl(gp_ctx* c, const gp_apps_wire* a, gp_algo algo, gp_mode mode, gp_results_wire* out) {
    gp_status s = check_args(c, a, algo, mode, out, "gp_pack_batch");
    if (s != GP_OK) return s;
    const int32_t q = a->n_apps;
    if (q == 0) return GP_OK;
    const auto t_begin = std::chrono::steady_clock::now();
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t es = a->quantity_bits == 64 ? 8 : 4;       // bytes per quantity
    const size_t os = out->node_bits == 16 ? 2 : 4;         // bytes per ExecutorNodes entry
    const int64_t* off = a->exec_out_off;                   // may be NULL: derived on the device, chunk bases summed here
    if (off) {
        const int64_t total = off[q];
        if (total < 0 || total > out->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, "gp_pack_batch: executor_nodes_cap too small");
        if (total > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, "gp_pack_batch: executor_nodes is NULL");
    }
    const size_t bq = es * (size_t)q, b32 = sizeof(int32_t) * (size_t)q;
    // the quantity columns are staged in ONE pitched device block (rows: drv cpu, drv mem, exe cpu, exe mem, drv gpu,
    // exe gpu) so that equally spaced host columns can be moved by a single 2-D DMA per chunk
    const size_t dpitch = (bq + 255) & ~(size_t)255;
    GP_CUDA(c, c->a_rows.reserve(dpitch * 6));
    GP_CUDA(c, c->a_count.reserve(b32));
    if (off) GP_CUDA(c, c->a_off.reserve(sizeof(int64_t) * (size_t)(q + 1)));
    GP_CUDA(c, c->r_driver.reserve(b32));
    GP_CUDA(c, c->r_exec.reserve(os * (size_t)(out->executor_nodes_cap + 1)));
    if (a->group) GP_CUDA(c, c->a_group.reserve(b32));
    if (a->skip_if_no_fit) GP_CUDA(c, c->a_skip.reserve((size_t)q));
    // Small batches are latency-bound: inputs are gathered by ONE kernel reading the mapped host buffers (every tiny
    // DMA copy of a chain pays its own fixed latency in stream order) and results are written straight into mapped host buffers.
    // Large ones are bandwidth-bound: DMA per pipelined chunk in both directions.
    const bool small = q <= kZeroCopyOutApps;
    void* mo_driver = small ? const_cast<void*>(mapped_ptr(c, out->driver_node, b32)) : nullptr;
    void* mo_exec = (small && out->executor_nodes) ? const_cast<void*>(mapped_ptr(c, out->executor_nodes, os * (size_t)out->executor_nodes_cap)) : nullptr;
    const bool out_mapped = small && mo_driver && (out->executor_nodes_cap == 0 || !out->executor_nodes || mo_exec);
    char* blk = c->a_rows.as<char>();
    DevApps dv{};
    const void* hq[6] = {a->drv_cpu, a->drv_mem, a->exe_cpu, a->exe_mem, a->drv_gpu, a->exe_gpu};    // staging row order
    dv.cols.q[0] = blk + 0 * dpitch; dv.cols.q[1] = blk + 1 * dpitch; dv.cols.q[3] = blk + 2 * dpitch; dv.cols.q[4] = blk + 3 * dpitch;
    dv.cols.q[2] = a->drv_gpu ? blk + 4 * dpitch : nullptr;
    dv.cols.q[5] = a->exe_gpu ? blk + 5 * dpitch : nullptr;
    dv.cols.count = c->a_count.as<int32_t>();
    dv.cols.group = a->group ? c->a_group.as<int32_t>() : nullptr;
    dv.cols.off = off ? c->a_off.as<int64_t>() : nullptr;
    dv.cols.bits = a->quantity_bits; dv.cols.mem_shift = a->mem_shift;
    dv.skip = a->skip_if_no_fit ? c->a_skip.as<uint8_t>() : nullptr;
    dv.n = q;
    DevResults dr;
    dr.driver = out_mapped ? (int32_t*)mo_driver : c->r_driver.as<int32_t>();
    dr.exec = out_mapped ? mo_exec : c->r_exec.p;
    dr.cap = out->executor_nodes_cap;
    dr.node_bits = out->node_bits;

    // Independent decisions are chunked and the chunks rotate over kLanes streams, so the H2D of
    // chunk i+1, the kernels of chunk i and the D2H of chunk i-1 overlap (PCIe is full duplex).
    // FIFO modes are one sequential pass: a single chunk.
    int n_chunks = 1;
    if (mode == GP_MODE_INDEPENDENT && q >= 2 * c->chunk_apps) {
        n_chunks = (q + c->chunk_apps - 1) / c->chunk_apps;
        if (n_chunks > kMaxChunks) n_chunks = kMaxChunks;
    }
    int2* scratch = nullptr;
    s = pack_begin(c, q, algo, mode, out->executor_nodes_cap, !off, &scratch, st);
    if (s != GP_OK) return s;
    // per-kernel CUDA events are for gp_last_stats; the pipelined path is bound by how fast the host thread can issue
    // its ~10 calls per chunk, so it leaves them out (pack_kernel_ns / prep_kernel_ns then read 0)
    struct EvGuard { gp_ctx* c; ~EvGuard() { c->record_events = true; } } ev_guard{c};
    c->record_events = n_chunks == 1;
    GP_CUDA(c, cudaEventRecord(c->ev_ready, st));      // snapshot + zeroed counters are ready
    const bool timeline = c->trace >= 2 && !c->record_events;
    if (timeline) GP_CUDA(c, cudaEventRecord(c->ev_t0, st));
    int64_t e_run = 0;                                 // ExecutorNodes entries before the current chunk
    for (int ch = 0; ch < n_chunks; ++ch) {
        const int32_t lo = (int32_t)((int64_t)q * ch / n_chunks), hi = (int32_t)((int64_t)q * (ch + 1) / n_chunks);
        const size_t n = (size_t)(hi - lo);
        cudaStream_t ls = n_chunks == 1 ? st : c->lane[ch % gp_ctx::kLanes];
        // ---- inputs -> HBM (the copies need not wait for the snapshot layout; the kernels below do) ----------------------------------------------------------------------------------
        bool gathered = false;
        if (small && !a->skip_if_no_fit) {
            CopyJobs jobs{};
            bool ok = true;
            auto add = [&](const void* src, void* dst, size_t bytes) {
                if (!src || !bytes) return;
                const void* m = mapped_ptr(c, src, bytes);
                if (!m || jobs.n >= 8) { ok = false; return; }
                jobs.j[jobs.n++] = CopyJob{m, dst, bytes};
            };
            // all six quantity rows when they are one equally spaced block, else row by row (<= 8 jobs in total)
            add(a->drv_cpu, blk + 0 * dpitch, bq); add(a->drv_mem, blk + 1 * dpitch, bq);
            add(a->exe_cpu, blk + 2 * dpitch, bq); add(a->exe_mem, blk + 3 * dpitch, bq);
            if (a->drv_gpu) add(a->drv_gpu, blk + 4 * dpitch, bq);
            if (a->exe_gpu) add(a->exe_gpu, blk + 5 * dpitch, bq);
            add(a->exe_count, c->a_count.p, b32);
            if (a->group) add(a->group, c->a_group.p, b32);
            if (off && ok) { if (jobs.n < 8) add(off, c->a_off.p, sizeof(int64_t) * (size_t)(q + 1)); else ok = false; }
            if (ok) {
                gp_multi_copy<<<q <= 64 ? 1 : 32, 256, 0, ls>>>(jobs);
                GP_CUDA(c, cudaGetLastError());
                c->last.kernel_launches += 1;
                gathered = true;
            }
        }
        if (!gathered) {
            // quantity columns: one 2-D DMA when the host columns are equally spaced (one pinned block laid out
            // column after column, as the shim allocates it), else one DMA per column
            int ncols = 4;
            if (a->drv_gpu && a->exe_gpu) ncols = 6;
            const ptrdiff_t spitch = (const char*)hq[1] - (const char*)hq[0];
            bool spaced = spitch >= (ptrdiff_t)bq && spitch <= ((ptrdiff_t)1 << 30);   // cudaMemcpy2D pitch limit (maxPitch ~2 GiB)
            for (int k = 2; spaced && k < ncols; ++k) spaced = ((const char*)hq[k] - (const char*)hq[k - 1]) == spitch;
            if (spaced && cudaMemcpy2DAsync(blk + es * (size_t)lo, dpitch, (const char*)hq[0] + es * (size_t)lo, (size_t)spitch,
                                            es * n, (size_t)ncols, cudaMemcpyHostToDevice, ls) != cudaSuccess) {
                cudaGetLastError();      // not accepted as a 2-D copy after all: column by column
                spaced = false;
            }
            if (!spaced) {
                for (int k = 0; k < ncols; ++k)
                    GP_CUDA(c, cudaMemcpyAsync(blk + k * dpitch + es * (size_t)lo, (const char*)hq[k] + es * (size_t)lo, es * n,
                                               cudaMemcpyHostToDevice, ls));
            }
            if (ncols == 4) {   // gpu columns given one at a time
                if (a->drv_gpu) GP_CUDA(c, cudaMemcpyAsync(blk + 4 * dpitch + es * (size_t)lo, (const char*)a->drv_gpu + es * (size_t)lo, es * n, cudaMemcpyHostToDevice, ls));
                if (a->exe_gpu) GP_CUDA(c, cudaMemcpyAsync(blk + 5 * dpitch + es * (size_t)lo, (const char*)a->exe_gpu + es * (size_t)lo, es * n, cudaMemcpyHostToDevice, ls));
            }
            GP_CUDA(c, cudaMemcpyAsync(c->a_count.as<int32_t>() + lo, a->exe_count + lo, sizeof(int32_t) * n, cudaMemcpyHostToDevice, ls));
            if (off) GP_CUDA(c, cudaMemcpyAsync(c->a_off.as<int64_t>() + lo, off + lo, sizeof(int64_t) * (n + 1), cudaMemcpyHostToDevice, ls));
            if (a->group) GP_CUDA(c, cudaMemcpyAsync(c->a_group.as<int32_t>() + lo, a->group + lo, sizeof(int32_t) * n, cudaMemcpyHostToDevice, ls));
            if (a->skip_if_no_fit) GP_CUDA(c, cudaMemcpyAsync(c->a_skip.as<uint8_t>() + lo, a->skip_if_no_fit + lo, n, cudaMemcpyHostToDevice, ls));
        }
        if (timeline) GP_CUDA(c, cudaEventRecord(c->ev[ch][0], ls));       // inputs of this chunk are in HBM
        if (n_chunks > 1) GP_CUDA(c, cudaStreamWaitEvent(ls, c->ev_ready, 0));
        // ---- this chunk's ExecutorNodes range ------------------------------------------------------------------
        int64_t e0, e1;
        if (off) { e0 = off[lo]; e1 = off[hi]; }
        else {
            int64_t acc = 0;
            const int32_t* cnt = a->exe_count;
            for (int32_t i = lo; i < hi; ++i) acc += cnt[i] > 0 ? cnt[i] : 0;
            e0 = e_run; e1 = e_run + acc; e_run = e1;
            if (e1 > out->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, "gp_pack_batch: executor_nodes_cap too small");
            if (e1 > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, "gp_pack_batch: executor_nodes is NULL");
        }
        s = pack_device_range(c, dv, lo, hi, e0, algo, mode, dr, scratch, ls, ch);
        if (s != GP_OK) return s;
        if (timeline) GP_CUDA(c, cudaEventRecord(c->ev[ch][1], ls));       // kernels of this chunk done
        if (out_mapped) continue;
        GP_CUDA(c, cudaMemcpyAsync(out->driver_node + lo, dr.driver + lo, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ls));
        if (e1 > e0)
            GP_CUDA(c, cudaMemcpyAsync((char*)out->executor_nodes + os * (size_t)e0, (char*)dr.exec + os * (size_t)e0, os * (size_t)(e1 - e0),
                                       cudaMemcpyDeviceToHost, ls));
    }
    if (timeline) for (int ch = 0; ch < n_chunks; ++ch) GP_CUDA(c, cudaEventRecord(c->ev[ch][2], n_chunks == 1 ? st : c->lane[ch % gp_ctx::kLanes]));
    c->ev_chunks = c->record_events ? n_chunks : 0;
    const auto t_issued = std::chrono::steady_clock::now();
    if (n_chunks > 1) {
        for (int l = 0; l < gp_ctx::kLanes && l < n_chunks; ++l) {
            GP_CUDA(c, cudaEventRecord(c->ev_done[l], c->lane[l]));
            GP_CUDA(c, cudaStreamWaitEvent(st, c->ev_done[l], 0));
        }
    }
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (timeline) {
        for (int ch = 0; ch < n_chunks; ++ch) {
            float a = 0, b = 0, d = 0;
            cudaEventElapsedTime(&a, c->ev_t0, c->ev[ch][0]); cudaEventElapsedTime(&b, c->ev_t0, c->ev[ch][1]); cudaEventElapsedTime(&d, c->ev_t0, c->ev[ch][2]);
            std::fprintf(stderr, "[gangpack]   chunk %d: inputs in HBM at %.1f us, kernels done at %.1f us, results on the host at %.1f us\n", ch, a * 1e3, b * 1e3, d * 1e3);
        }
    }
    if (c->trace) {
        const auto t_done = std::chrono::steady_clock::now();
        std::fprintf(stderr, "[gangpack] pack_batch q=%d chunks=%d bits=%d/%d out_mapped=%d issue=%.1fus wait=%.1fus\n", q, n_chunks,
                     a->quantity_bits, out->node_bits, (int)out_mapped, std::chrono::duration<double, std::micro>(t_issued - t_begin).count(),
                     std::chrono::duration<double, std::micro>(t_done - t_issued).count());
    }
    // scan statistics stay on the device until gp_last_stats asks for them
    return host_error(c);
}

gp_status gp_pack_one(gp_ctx* c, gp_algo algo, int64_t drv_cpu, int64_t drv_mem, int64_t drv_gpu, int64_t exe_cpu,
                      int64_t exe_mem, int64_t exe_gpu, int32_t exe_count, int32_t* has_capacity, int32_t* driver_node,
                      int32_t* executor_nodes) {
    if (!enter(c)) return GP_ERR_INVALID;
    if (!has_capacity || !driver_node) return fail(c, GP_ERR_INVALID, "gp_pack_one: NULL outputs");
    if (exe_count > 0 && !executor_nodes) return fail(c, GP_ERR_INVALID, "gp_pack_one: executor_nodes is NULL");
    // The tuple and the result travel through a context-owned mapped pinned block: no DMA copies at all
    // on this latency-critical path (one app = one SparkBinPackFunction call).
    const size_t n_exec = exe_count > 0 ? (size_t)exe_count : 0;
    const size_t need = 128 + sizeof(int32_t) * (n_exec + 1);
    if (need > c->one_bytes) {
        GP_CUDA(c, cudaSetDevice(c->device));
        if (c->one_block) { gp_free_pinned(c, c->one_block); c->one_block = nullptr; c->one_bytes = 0; }
        void* blk = nullptr;
        gp_status st = gp_alloc_pinned(c, need * 2, &blk);
        if (st != GP_OK) return st;
        c->one_block = blk; c->one_bytes = need * 2;
    }
    int64_t* q = static_cast<int64_t*>(c->one_block);         // [0..5] tuple, [6..7] offsets
    q[0] = drv_cpu; q[1] = drv_mem; q[2] = drv_gpu; q[3] = exe_cpu; q[4] = exe_mem; q[5] = exe_gpu;
    q[6] = 0; q[7] = (int64_t)n_exec;
    int32_t* i32 = reinterpret_cast<int32_t*>(q + 8);          // [0] count, [1] driver result
    i32[0] = exe_count; i32[1] = -1;
    int32_t* exec_out = reinterpret_cast<int32_t*>(static_cast<char*>(c->one_block) + 128);
    gp_apps a{};
    a.n_apps = 1;
    a.drv_cpu_milli = q + 0; a.drv_mem_bytes = q + 1; a.drv_gpu = q + 2;
    a.exe_cpu_milli = q + 3; a.exe_mem_bytes = q + 4; a.exe_gpu = q + 5;
    a.exe_count = i32;
    a.exec_out_off = algo == GP_MINIMAL_FRAGMENTATION ? q + 6 : nullptr;   // derived on the device where the kernel can
    gp_results r{};
    r.driver_node = i32 + 1;
    r.executor_nodes = exec_out;
    r.executor_nodes_cap = (int64_t)n_exec;
    gp_status s = gp_pack_batch(c, &a, algo, GP_MODE_INDEPENDENT, &r);
    if (s != GP_OK) return s;
    const int32_t d = i32[1];
    *has_capacity = d >= 0 ? 1 : 0;
    *driver_node = d >= 0 ? d : -1;
    if (d >= 0 && n_exec) std::memcpy(executor_nodes, exec_out, sizeof(int32_t) * n_exec);
    return GP_OK;
}

}  // extern "C"

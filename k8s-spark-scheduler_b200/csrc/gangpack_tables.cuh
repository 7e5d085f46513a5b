// gangpack_tables.cuh -- independent mode (GP_MODE_INDEPENDENT) for tightly-pack / distribute-evenly:
// per-executor-shape capacity tables + the fused (prep + pack) warp-per-application kernel.
//
// Reference semantics (all under /root/reference; LIB = vendor/github.com/palantir/k8s-spark-scheduler-lib/pkg):
//   SparkBinPack driver loop        LIB/binpack/binpack.go:60-87
//   tightlyPackExecutors            LIB/binpack/pack_tightly.go:34-63
//   distributeExecutorsEvenly       LIB/binpack/distribute_evenly.go:34-73
//   node capacity                   LIB/capacity/capacity.go:36-75
//
// Why tables.  Every application of an independent batch is packed against the SAME snapshot
// (internal/extender/unschedulablepods.go:132-166; each Predicate's own pack, resource.go:321), and a node's executor
// capacity depends only on the executor request -- the "shape" (cpu, mem, gpu).  Real queues hold few shapes (the
// synthetic one: 12).  So instead of every application re-scanning the node order, each distinct shape is scanned ONCE.
// The three dependent phases run in ONE persistent launch, gp_decide_tables, as ticket-ordered work items (see there):
//   1 gp_classify_apps    thread per application: intern its shape in a small hash table (atomicCAS on a 64-bit
//                         fingerprint; the full tuple is verified again by the consumer, so a fingerprint collision costs
//                         a fallback, never a wrong answer) and derive the ExecutorNodes offsets when the caller gave none
//                         (decoupled look-back over the tiles);
//   2 gp_build_shape_tables  one item per kTabSeg-node segment of one (shape, instance group): every thread evaluates 4
//                         consecutive nodes, a block-wide scan plus a look-back over the earlier segments of the same
//                         (shape, group) turns capacities into the prefix table
//                                       S[i] = sum_{n<i} min(cap(n|0), CLAMP)   (tightly-pack) or
//                                       M[i] = #{n<i : cap(n|0) >= 1}            (distribute-evenly),
//                         and the first kPlaceLen entries of the driver-free placement P[t] = node of the t-th executor;
//                         one item per (driver shape, instance group) finds the first driver candidate the shape fits on;
//   3 decide              ONE THREAD per application (with the tables a decision is O(log N + k) scalar work -- a warp per
//                         application, right for an O(N) scan, would idle 31 lanes): feasibility is
//                         S[ne] - delta(d) >= k  per driver candidate d starting at the shape's first fit (delta = what the
//                         driver displaces on its own node: O(1) per candidate, the reference's loop binpack.go:67-85
//                         verbatim).  ExecutorNodes is P shifted by delta past the driver's run, written by the whole warp
//                         with coalesced stores, when its largest index k - 1 + delta is below kPlaceLen; otherwise it is
//                         emitted by walking the table from the shape's first hosting node (one word per (shape, group),
//                         written by phase 2) with the next word always in flight (zero-capacity runs are jumped by a galloping
//                         search).
// What the tables cannot answer exactly -- more than kMaxShapes distinct shapes in a batch, executor counts above the table
// clamp, distribute-evenly placements that need more than one round -- is appended, already prepared (PrepApp), to a list
// that the warp-per-application scan kernel gp_pack_listed (the node-order scan of gangpack_kernels.cuh) works off.
// GANGPACK_TABLES=0 sends every application down that path.
#pragma once

#include "gangpack_kernels.cuh"

namespace gp {

constexpr int kShapeSlots = 1024;     // hash slots (power of two)
constexpr int kShapeProbes = 16;      // linear probes before giving up (-> scan path)
constexpr int kMaxShapes = 64;        // dense tables per batch
constexpr int kPlaceLen = 256;        // placement prefix per (shape, group): covers every count <= 128 whatever the driver takes

struct __align__(16) ShapeEntry {     // 96 bytes
    unsigned long long key;           // fingerprint, never 0; 0 = empty (claimed with atomicCAS)
    int32_t id;                       // dense table id in claim order; -1: more than kMaxShapes shapes in this batch
    uint32_t flags;                   // bit0: gpu request != 0
    DimDiv div[3];                    // executor cpu, mem, gpu: the request itself (div[t].e) and how to divide by it
};
static_assert(sizeof(ShapeEntry) == 96, "ShapeEntry layout");

struct __align__(16) DriverEntry {    // 48 bytes: interned driver request
    unsigned long long key;
    int32_t id;
    uint32_t pad;
    int64_t d[3];
    int64_t pad2;
};
static_assert(sizeof(DriverEntry) == 48, "DriverEntry layout");

// device-side header of one table set.  The counters, the hash keys and the look-back words are zero when a call starts:
// the buffer is zeroed when it is allocated, and gp_pack_listed, the last kernel of every call, zeroes what the call used
// (n_listed excepted: gp_pack_listed reads it, and the first classify tile of the next call zeroes it).
struct ShapeHeader {
    int32_t n_shapes;                 // executor shapes claimed so far (may exceed kMaxShapes)
    int32_t n_dshapes;                // driver shapes claimed so far
    int32_t n_listed;                 // applications handed to the scan kernel
    int32_t pad;
    int32_t id_slot[kMaxShapes];      // dense executor-shape id -> hash slot
    int32_t did_slot[kMaxShapes];     // dense driver-shape id -> hash slot
    uint32_t ticket;                  // next work item of gp_decide_tables
    uint32_t cls_done;                // classify tiles finished
    uint32_t tab_done;                // table items finished
    uint32_t dec_next;                // decide chunks claimed past the grid's warp count (the first chunk of a warp is fixed)
};
static_assert(sizeof(ShapeHeader) <= 1024, "ShapeHeader");

struct ShapeTables {
    ShapeEntry* entries;              // [kShapeSlots]
    DriverEntry* dentries;            // [kShapeSlots]
    ShapeHeader* hdr;
    unsigned long long* cls_status;   // [classify tiles] look-back words of the derived offsets (zero at the start of a call)
    unsigned long long* seg_status;   // [kMaxShapes * segments] look-back words of the table segments (zero at the start of a call)
    const int32_t* seg_pre;           // [n_groups + 1] table segments before each group (the snapshot's, gp_build_slots_drv)
    uint32_t* table;                  // [kMaxShapes][pitch] exclusive prefix per instance group, indexed by slot
    uint32_t* total;                  // [kMaxShapes][n_groups]
    int32_t* firstfit;                // [kMaxShapes][n_groups] first driver-order position the driver shape fits on (nd: none)
    int32_t* first_host;              // [kMaxShapes][n_groups] first executor-order position with capacity > 0 for the shape (ne: none)
    int32_t* place;                   // [kMaxShapes][n_groups][kPlaceLen] node receiving the t-th executor without a driver
                                      // (entries t >= the group's total are not written)
    int32_t pitch;                    // row length (>= n_slots, multiple of 4)
    int32_t n_groups;
};

// largest executor count / per-node capacity the uint32 prefix of a group can carry without wrapping
__device__ __forceinline__ uint32_t table_clamp(int32_t ne) {
    const uint32_t by_len = 0xFFFFFFFFu / (uint32_t)(ne > 0 ? ne : 1);
    return by_len < (uint32_t)kMaxCount ? by_len : (uint32_t)kMaxCount;
}

// ---------------------------------------------------------------------------------------------------------------
// cross-CTA signalling inside the one launch
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Polling back-off cap (ns) of the phase waits and the look-back.  A waiter notices a completion up to one sleep late,
// and a phase hand-off is on the critical path of the whole launch; one poller per CTA (per warp in the look-back) keeps
// the polling traffic small even at this cap.
constexpr unsigned kPollMaxNs = 128;
// thread 0 of a CTA: wait until *ctr >= n (acquire: the producers' writes are visible to the whole CTA after the
// __syncthreads that follows)
__device__ __forceinline__ void wait_count(const uint32_t* ctr, uint32_t n) {
    unsigned ns = 32;
    while (ld_acquire_u32(ctr) < n) { __nanosleep(ns); if (ns < kPollMaxNs) ns <<= 1; }
    __threadfence();
}
// ---- phase timeline of gp_decide_tables (diagnostic build, -DGP_DECIDE_TIMELINE; tools/decide_timeline.py) ----------
// Thread 0 of every CTA stamps %globaltimer when it claims a ticket and when the item is counted done, and when its
// cls_done / tab_done waits return; every warp stamps the start and end of its decide chunks.  Each CTA and warp writes
// its own slots (no shared counter that would itself serialise), and each launch overwrites the previous one's.  The
// shipped build compiles none of this.
#ifdef GP_DECIDE_TIMELINE
enum TlKind : uint32_t { kTlCls = 0, kTlSeg = 1, kTlFirstFit = 2, kTlClsWait = 3, kTlTabWait = 4 };
constexpr int kTlCtas = 1024;           // CTAs recorded
constexpr int kTlPerCta = 48;           // records per CTA (further ones are counted, not stored)
constexpr int kTlWarps = kTlCtas * (kTabThreads / 32);
struct TlRec { unsigned long long t0, t1; uint32_t kind, item, pad0, pad1; };     // t0: claim / wait start, t1: done / return
struct TlBuf {
    uint32_t grid, n_cls, n_tab, n_chunks;
    uint32_t n[kTlCtas];
    TlRec rec[kTlCtas][kTlPerCta];
    unsigned long long warp[kTlWarps][2];                    // first decide chunk starts, last one ends (0: no chunk)
    uint32_t warp_chunks[kTlWarps];
};
__device__ TlBuf g_tl;
__device__ __forceinline__ unsigned long long tl_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void tl_rec(uint32_t& n, uint32_t kind, uint32_t item, unsigned long long t0) {
    if (blockIdx.x < kTlCtas && n < kTlPerCta) g_tl.rec[blockIdx.x][n] = TlRec{t0, tl_now(), kind, item, 0u, 0u};
    ++n;
}
#define GP_TL(...) __VA_ARGS__
#else
#define GP_TL(...)
#endif

// whole CTA after writing an item's output: count it done (release)
__device__ __forceinline__ void signal_done(uint32_t* ctr) {
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); atomicAdd(ctr, 1u); }
}

// Look-back status word of a scanned item (classify tile, table segment): flag in bits 62-63, value below.
constexpr unsigned long long kStAggregate = 1ull << 62;     // the item's own sum is published
constexpr unsigned long long kStInclusive = 2ull << 62;     // the sum of every item of the chain up to and including it
constexpr unsigned long long kStValue = (1ull << 62) - 1;

// Decoupled look-back (Merrill & Garland 2016), called by one whole warp: the exclusive prefix of item `idx` of the chain
// of status words [first, idx), idx > first.  Item `first` always publishes an inclusive word, so the walk ends there.
// Every item it waits for has a smaller ticket (see gp_decide_tables).
__device__ __forceinline__ unsigned long long lookback(const unsigned long long* status, int32_t first, int32_t idx, int lane) {
    unsigned long long excl = 0;
    for (int32_t end = idx;; end -= 32) {
        const int32_t j = end - 1 - lane;                   // lane 0: the nearest predecessor
        unsigned long long v = kStInclusive;                // before the chain: an inclusive 0
        if (j >= first) {
            unsigned ns = 32;
            while (((v = ld_relaxed_u64(status + j)) >> 62) == 0) { __nanosleep(ns); if (ns < kPollMaxNs) ns <<= 1; }
        }
        const unsigned inc = __ballot_sync(kFull, (v >> 62) == 2);
        const int stop = inc ? __ffs(inc) - 1 : 31;         // nearest inclusive word: nothing beyond it is needed
        unsigned long long add = lane <= stop ? (v & kStValue) : 0ull;
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) add += __shfl_xor_sync(kFull, add, d);
        excl += add;
        if (inc) return excl;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// phase 1 (classify): intern executor and driver shapes, derive offsets -- one tile of kTabThreads applications
// ---------------------------------------------------------------------------------------------------------------
// intern one request tuple (fingerprint fp) into the open-addressing table of ENTRY records; returns the slot or -1.
// `init(entry, slot)` fills a freshly claimed entry.  Called by ONE lane per distinct fingerprint of a warp.
template <class ENTRY, class INIT>
__device__ __forceinline__ int32_t intern_shape(ENTRY* table, unsigned long long fp, INIT init) {
    int32_t slot = (int32_t)(fp & (kShapeSlots - 1));
    for (int p = 0; p < kShapeProbes; ++p) {
        ENTRY* en = table + slot;
        // plain (L1-cacheable) load: a key never changes once set, and a stale 0 is resolved by the CAS below
        unsigned long long cur = en->key;
        if (cur == 0) {
            cur = atomicCAS(&en->key, 0ull, fp);
            if (cur == 0) { init(en, slot); cur = fp; }
        }
        if (cur == fp) return slot;
        slot = (slot + 1) & (kShapeSlots - 1);
    }
    return -1;
}

struct OneScratch {
    unsigned long long part[kTabThreads / 32];
    unsigned long long base;
    uint32_t ticket;
    int32_t first_host;
};

// ExecutorNodes offsets = exclusive prefix sum of max(count, 0), when the caller passed none: a block scan of the tile +
// the sum of every tile before it, by look-back over the tiles in ticket order
__device__ __forceinline__ void classify_offsets(OneScratch& sh, int32_t tile, int32_t n_apps, const AppColumns& cols,
                                                 const ShapeTables& tabs, int64_t off_base, int64_t* off_out) {
    const int32_t i = tile * kTabThreads + (int32_t)threadIdx.x;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int32_t mine = (i < n_apps) ? max(cols.count[i], 0) : 0;
    const uint32_t incl = warp_incl_scan((uint32_t)mine, lane);
    unsigned long long wsum = (unsigned long long)mine;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) wsum += __shfl_xor_sync(kFull, wsum, d);
    if (lane == 31) sh.part[w] = incl;
    __shared__ unsigned long long s_wsum[kTabThreads / 32];
    if (lane == 0) s_wsum[w] = wsum;
    __syncthreads();
    if (w == 0) {
        unsigned long long agg = lane < kTabThreads / 32 ? s_wsum[lane] : 0ull;
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) agg += __shfl_xor_sync(kFull, agg, d);
        unsigned long long excl = 0;
        if (tile == 0) {
            if (lane == 0) st_relaxed_u64(tabs.cls_status, kStInclusive | agg);
        } else {
            if (lane == 0) st_relaxed_u64(tabs.cls_status + tile, kStAggregate | agg);
            excl = lookback(tabs.cls_status, 0, tile, lane);
            if (lane == 0) st_relaxed_u64(tabs.cls_status + tile, kStInclusive | ((excl + agg) & kStValue));
        }
        if (lane == 0) sh.base = excl;
    }
    __syncthreads();
    unsigned long long base = (unsigned long long)off_base + sh.base, prev = 0;
    for (int t = 0; t < w; ++t) prev += sh.part[t];
    if (i < n_apps) off_out[i] = (int64_t)(base + prev + incl - (uint32_t)mine);
    if (i == n_apps - 1) off_out[n_apps] = (int64_t)(base + prev + incl);
}

// per thread: today's gp_classify_apps body
// It reads nothing of the snapshot: gp_decide_tables runs it before the slot layout has ended.
__device__ __forceinline__ void gp_classify_apps(int32_t tile, int32_t n_apps, const AppColumns& cols, const ShapeTables& tabs,
                                                 int32_t* app_slot) {
    const int32_t i = tile * kTabThreads + (int32_t)threadIdx.x;
    const int lane = threadIdx.x & 31;
    const unsigned act = __ballot_sync(kFull, i < n_apps);     // the lanes that intern (the whole warp except in the last tile)
    if (i >= n_apps) return;

    // A queue has few distinct requests: the lanes of a warp that carry the same fingerprint elect ONE of them to probe /
    // claim the entry (100 000 threads doing their own CAS on a dozen lines serialise on those lines); the consumer
    // verifies the full tuple, so a fingerprint collision inside a warp only sends an application to the scan.
    const int64_t e0 = cols.load(3, i), e1 = cols.load(4, i), e2 = cols.load(5, i);
    const bool e_ok = e0 >= 0 && e1 >= 0 && e2 >= 0 && e0 < kMaxQuantity && e1 < kMaxQuantity && e2 < kMaxQuantity;
    const unsigned long long efp = e_ok ? shape_fingerprint(e0, e1, e2) : 0ull;
    {
        const unsigned same = __match_any_sync(act, efp);
        const int leader = __ffs(same) - 1;
        int32_t found = -1;
        if (lane == leader && e_ok)
            found = intern_shape(tabs.entries, efp, [&](ShapeEntry* en, int32_t slot) {
                // this lane owns the entry: dense id, division recipes (verified by every consumer against its own tuple).
                // A recipe depends on the request alone; prep_dim's max_avail only decides `fast`, which is not kept here.
                int32_t id = atomicAdd(&tabs.hdr->n_shapes, 1);
                if (id >= kMaxShapes) id = -1;
                int bad = 0; uint64_t l; bool fast = true;
                en->div[0] = prep_dim(0, e0, 0, 0, bad, l, fast);
                en->div[1] = prep_dim(0, e1, 1, 0, bad, l, fast);
                en->div[2] = prep_dim(0, e2, 2, 0, bad, l, fast);
                en->flags = e2 != 0 ? 1u : 0u;
                en->id = id;
                if (id >= 0) tabs.hdr->id_slot[id] = slot;
            });
        app_slot[i] = __shfl_sync(act, found, leader);
    }

    // ---- the driver request, interned the same way: its first fitting candidate is searched once per shape ----------
    const int64_t d0 = cols.load(0, i), d1 = cols.load(1, i), d2 = cols.load(2, i);
    const bool d_ok = d0 >= 0 && d1 >= 0 && d2 >= 0 && d0 < kMaxQuantity && d1 < kMaxQuantity && d2 < kMaxQuantity;
    const unsigned long long dfp = d_ok ? shape_fingerprint(d0 ^ 0x5bd1e995, d1, d2) : 0ull;
    {
        const unsigned same = __match_any_sync(act, dfp);
        const int leader = __ffs(same) - 1;
        int32_t dfound = -1;
        if (lane == leader && d_ok)
            dfound = intern_shape(tabs.dentries, dfp, [&](DriverEntry* en, int32_t slot) {
                int32_t id = atomicAdd(&tabs.hdr->n_dshapes, 1);
                if (id >= kMaxShapes) id = -1;
                en->d[0] = d0; en->d[1] = d1; en->d[2] = d2;
                en->id = id;
                if (id >= 0) tabs.hdr->did_slot[id] = slot;
            });
        app_slot[n_apps + i] = __shfl_sync(act, dfound, leader);         // second half of the array: driver-shape slots
    }
}

// ---------------------------------------------------------------------------------------------------------------
// phase 2 (tables): capacity prefix of one segment of one (shape, instance group)
// ---------------------------------------------------------------------------------------------------------------
// Segment `seg` of `n_seg` covers executor-order positions [seg * kTabSeg, min(+kTabSeg, ne)) of group `grp`; every
// thread evaluates kTabPerThread consecutive nodes.  `st` is the segment's look-back status word; the chain of the
// (shape, group) is st - seg .. st - seg + n_seg - 1.  Together the segments write
//     S[i] = sum_{n<i} min(cap(n|0), CLAMP)   (tightly-pack) or   M[i] = #{n<i : cap(n|0) >= 1}   (distribute-evenly),
// total = S[ne], first_host (first position with capacity, ne: none) and the placement prefix P[t < min(total, kPlaceLen)].
template <int ALGO>
__device__ __forceinline__ void gp_build_shape_tables(OneScratch& sh, const Snapshot& s, const ShapeTables& tabs, int id, int grp,
                                                      int32_t seg, int32_t n_seg, unsigned long long* st) {
    const ShapeEntry& en = tabs.entries[tabs.hdr->id_slot[id]];
    const DimDiv dc = en.div[0], dm = en.div[1], dg = en.div[2];
    const bool ug = (en.flags & 1u) || (s.meta->flags & kSnapGpuNegative);
    const GroupDesc g = s.groups[grp];
    const int32_t ne = g.ne;
    const uint32_t clamp = table_clamp(ne);
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const longlong2* gpair = s.pair + g.sbase;
    const int64_t* ggpu = s.gpu + g.sbase;
    uint32_t* out = tabs.table + (size_t)id * tabs.pitch + g.sbase;
    int32_t* place = tabs.place + ((size_t)id * tabs.n_groups + grp) * kPlaceLen;

    const int32_t i0 = seg * kTabSeg + tid * kTabPerThread;
    uint32_t v[kTabPerThread];
    uint32_t sum = 0;
    int32_t my_first = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < kTabPerThread; ++j) {
        const int32_t i = i0 + j;
        uint32_t c = 0;
        if (i < ne) {
            const longlong2 a = __ldg(gpair + i);
            c = min(cap_dim(a.x, dc, clamp), cap_dim(a.y, dm, clamp));
            if (ug) c = min(c, cap_dim(__ldg(ggpu + i), dg, clamp));
            if (ALGO == 1) c = c != 0 ? 1u : 0u;
        }
        if (c != 0 && i < my_first) my_first = i;
        v[j] = sum;             // exclusive within the thread
        sum += c;
    }
    // block-wide exclusive scan of the per-thread sums, and the segment's first hosting node
    if (tid == 0) sh.first_host = 0x7fffffff;
    const uint32_t incl = warp_incl_scan(sum, lane);
    if (lane == 31) sh.part[w] = incl;
    __syncthreads();
    {
        const uint32_t wmin = __reduce_min_sync(kFull, (uint32_t)my_first);
        if (lane == 0 && wmin != 0x7fffffffu) atomicMin(&sh.first_host, (int32_t)wmin);
    }
    uint32_t before = 0, seg_total = 0;
    for (int t = 0; t < kTabThreads / 32; ++t) { if (t < w) before += (uint32_t)sh.part[t]; seg_total += (uint32_t)sh.part[t]; }
    if (w == 0) {               // the segment's base: the sum of the segments before it in the same (shape, group)
        unsigned long long base = 0;
        if (seg == 0) {
            if (lane == 0) st_relaxed_u64(st, kStInclusive | seg_total);
        } else {
            if (lane == 0) st_relaxed_u64(st, kStAggregate | seg_total);
            base = lookback(st - seg, 0, seg, lane);
            if (lane == 0) st_relaxed_u64(st, kStInclusive | (base + seg_total));
        }
        if (lane == 0) sh.base = base;
    }
    __syncthreads();
    const uint32_t seg_base = (uint32_t)sh.base;
    const uint32_t base = seg_base + before + incl - sum;
    if (i0 + kTabPerThread <= ne && ((g.sbase + i0) & 3) == 0) {
        *reinterpret_cast<uint4*>(out + i0) = make_uint4(base + v[0], base + v[1], base + v[2], base + v[3]);
    } else {
#pragma unroll
        for (int j = 0; j < kTabPerThread; ++j) if (i0 + j < ne) out[i0 + j] = base + v[j];
    }
    // placement prefix: a node whose first executor index is below kPlaceLen writes its run [S, min(S + c, kPlaceLen))
    // (the (shape, group) writes at most kPlaceLen words in all; only the first hosting nodes of the order do anything)
    if (base < (uint32_t)kPlaceLen) {
#pragma unroll
        for (int j = 0; j < kTabPerThread; ++j) {
            const uint32_t p0 = base + v[j];
            const uint32_t p1 = base + (j + 1 < kTabPerThread ? v[j + 1] : sum);
            if (p0 < p1 && p0 < (uint32_t)kPlaceLen) {
                const int32_t node = __ldg(s.slot_node + g.sbase + i0 + j);
                const uint32_t end = p1 < (uint32_t)kPlaceLen ? p1 : (uint32_t)kPlaceLen;
                for (uint32_t t = p0; t < end; ++t) place[t] = node;
            }
        }
    }
    // first_host: the one segment with nothing before it and something in it (or the last one, when the group hosts none);
    // total: the last segment
    if (tid == 0) {
        const size_t at = (size_t)id * tabs.n_groups + grp;
        if (seg_base == 0 && seg_total != 0) tabs.first_host[at] = sh.first_host;
        if (seg == n_seg - 1) {
            tabs.total[at] = seg_base + seg_total;
            if (seg_base + seg_total == 0) tabs.first_host[at] = ne;
        }
    }
}

// phase 2 (tables): first fitting driver candidate per (driver shape, instance group)
__device__ __forceinline__ void driver_firstfit_block(const Snapshot& s, const ShapeTables& tabs, int id, int grp) {
    __shared__ int32_t s_first;
    const DriverEntry& en = tabs.dentries[tabs.hdr->did_slot[id]];
    const int64_t d0 = en.d[0], d1 = en.d[1], d2 = en.d[2];
    const GroupDesc g = s.groups[grp];
    const bool ug = d2 != 0 || (s.meta->flags & kSnapGpuNegative);
    const longlong2* gpair = s.pair + g.sbase;
    const int64_t* ggpu = s.gpu + g.sbase;
    if (threadIdx.x == 0) s_first = g.nd;
    __syncthreads();
    // kFitPerThread independent candidates per thread and step: a shape that fits late walks the order in few dependent
    // load round trips
    constexpr int kFitPerThread = 8;
    for (int32_t j0 = 0; j0 < g.nd; j0 += kFitPerThread * kTabThreads) {
        int32_t ls[kFitPerThread];
#pragma unroll
        for (int u = 0; u < kFitPerThread; ++u) {
            const int32_t j = j0 + u * kTabThreads + (int32_t)threadIdx.x;
            ls[u] = j < g.nd ? s.drv_slot[g.dbase + j] : -1;
        }
        int32_t mine = 0x7fffffff;
#pragma unroll
        for (int u = 0; u < kFitPerThread; ++u) {
            if (ls[u] < 0) continue;
            const longlong2 v = __ldg(gpair + ls[u]);
            // driverResources.GreaterThan(available) == false
            const bool fits = !(d0 > v.x) && !(d1 > v.y) && !(ug && d2 > __ldg(ggpu + ls[u]));
            if (fits && mine == 0x7fffffff) mine = j0 + u * kTabThreads + (int32_t)threadIdx.x;
        }
        if (mine != 0x7fffffff) atomicMin(&s_first, mine);
        __syncthreads();
        if (s_first < g.nd) break;               // block-uniform
    }
    if (threadIdx.x == 0) tabs.firstfit[(size_t)id * tabs.n_groups + grp] = s_first;
}

// ---------------------------------------------------------------------------------------------------------------
// phase 3 (decide): one thread per application
// ---------------------------------------------------------------------------------------------------------------
// The tables are written earlier in the same launch: every load of them below is an ordinary (coherent) load, never the
// read-only path.
// prefix value S(i), i in [0, ne]
__device__ __forceinline__ uint32_t tab_at(const uint32_t* tab, int32_t i, int32_t ne, uint32_t total) {
    return i < ne ? tab[i] : total;
}
// smallest p in (lo, ne] with S(p) > val; requires S(ne) = total > val
__device__ __forceinline__ int32_t tab_next_above(const uint32_t* tab, int32_t lo, int32_t ne, uint32_t total, uint32_t val,
                                                  unsigned long long& probes) {
    int32_t a = lo + 1, b = ne;                     // answer in [a, b], S(b) > val
    // gallop first: the zero-capacity runs inside a walk are short (1-2 probes instead of log2(ne))
    int32_t step = 1;
    while (a < b) {
        const int32_t t = a + step - 1 < b - 1 ? a + step - 1 : b - 1;      // t in [a, b-1]
        ++probes;
        if (tab_at(tab, t, ne, total) > val) { b = t; break; }             // answer in [a, t]
        a = t + 1;                                                          // answer in [t+1, b]
        step <<= 1;
    }
    while (a < b) {
        const int32_t mid = (a + b) >> 1;
        if (tab_at(tab, mid, ne, total) > val) b = mid; else a = mid + 1;
        ++probes;
    }
    return a;
}

// What the decide phase reads of one application before the tables exist: its columns, the validation, and the shape
// slots phase 1 interned (with their full tuples checked).  Everything here was written before cls_done, so a warp loads
// it while its CTA still waits for tab_done, and the decision itself starts from the table loads.
struct AppIn {
    int64_t d[3];                     // driver request
    int64_t off;                      // ExecutorNodes offset
    int32_t k, grp;                   // executor count, instance group
    int32_t slot;                     // executor-shape hash slot whose table decides; -1: the scan decides
    int32_t did;                      // dense driver-shape id with this exact request; -1: the driver loop starts at 0
    int32_t bad;                      // validation error bits
    bool live;                        // i < n_apps
};
__device__ __forceinline__ AppIn decide_load(int32_t i, const Snapshot& s, const AppColumns& cols, const ShapeTables& tabs,
                                             const int32_t* app_slot, int32_t n_apps, int64_t out_cap, int force_scan) {
    AppIn a;
    a.live = i < n_apps;
    a.d[0] = a.d[1] = a.d[2] = 0; a.off = 0; a.k = 0; a.grp = 0; a.slot = -1; a.did = -1; a.bad = 0;
    if (!a.live) return a;
    const int64_t d_cpu = cols.load(0, i), d_mem = cols.load(1, i), d_gpu = cols.load(2, i);
    const int64_t e_cpu = cols.load(3, i), e_mem = cols.load(4, i), e_gpu = cols.load(5, i);
    const int32_t kk = cols.count[i];
    const int32_t grp = cols.group ? cols.group[i] : 0;
    const int64_t off = cols.off[i], off1 = cols.off[i + 1];
    // ---- validation (types.SparkApplicationResources must be non-negative and inside the exact-int64 domain) ----
    int bad = 0;
    if (d_cpu < 0 || d_mem < 0 || d_gpu < 0 || e_cpu < 0 || e_mem < 0 || e_gpu < 0 || kk < 0) bad |= kErrNegativeRequest;
    if (d_cpu >= kMaxQuantity || d_mem >= kMaxQuantity || d_gpu >= kMaxQuantity || e_cpu >= kMaxQuantity || e_mem >= kMaxQuantity ||
        e_gpu >= kMaxQuantity || kk > kMaxCount) bad |= kErrUnrepresentable;
    if (grp < 0 || grp >= s.n_groups) bad |= kErrBadGroup;
    if (off < 0 || off1 - off != (int64_t)(kk > 0 ? kk : 0) || off1 > out_cap) bad |= kErrBadOffsets;
    a.d[0] = d_cpu; a.d[1] = d_mem; a.d[2] = d_gpu; a.off = off; a.k = kk; a.grp = grp; a.bad = bad;
    if (bad || force_scan) return a;
    const int32_t slot = app_slot[i];
    if (slot >= 0) {
        const ShapeEntry* en = tabs.entries + slot;         // the full tuple decides, not the fingerprint
        if (en->id >= 0 && en->div[0].e == e_cpu && en->div[1].e == e_mem && en->div[2].e == e_gpu &&
            (uint32_t)kk <= table_clamp(s.groups[grp].ne)) a.slot = slot;
    }
    const int32_t ds = app_slot[n_apps + i];
    if (ds >= 0) {
        const DriverEntry& de = tabs.dentries[ds];
        if (de.id >= 0 && de.d[0] == d_cpu && de.d[1] == d_mem && de.d[2] == d_gpu) a.did = de.id;
    }
    return a;
}

// i: the application of this lane, a: what decide_load read of it.  Applications the tables cannot decide are prepared
// (PrepApp) and appended to `listed`; force_scan appends every application.
template <int ALGO, class OUT>
__device__ __forceinline__ void decide_app(int32_t i, const AppIn& a, const Snapshot& s, const AppColumns& cols,
                                            const ShapeTables& tabs, int32_t* __restrict__ driver_node,
                                            OUT* __restrict__ executor_nodes, PrepApp* __restrict__ prep,
                                            int32_t* __restrict__ listed, int* __restrict__ err, volatile int* __restrict__ err_host,
                                            unsigned long long& probes, unsigned long long& drivers) {
    const int lane = threadIdx.x & 31;
    // this lane's share of the warp's coalesced emission (sh_k = 0: none): out[sh_dst + t] = place[sh_src + shifted t]
    uint32_t sh_k = 0, sh_cut = 0, sh_delta = 0;
    int64_t sh_dst = 0, sh_src = 0;
    if (a.live) {
        const int64_t d_cpu = a.d[0], d_mem = a.d[1], d_gpu = a.d[2];
        const int32_t kk = a.k, grp = a.grp;
        const int64_t off = a.off;
        if (a.bad) {
            atomicOr(err, a.bad); *err_host = a.bad;
            driver_node[i] = -1;
        } else {
            const GroupDesc g = s.groups[grp];
            const int32_t ne = g.ne, nd = g.nd;
            const uint32_t k = (uint32_t)kk;
            const int snap_flags = s.meta->flags;
            bool need_scan = a.slot < 0;
            int32_t result = -1;
            const ShapeEntry* en = nullptr;
            const uint32_t* tab = nullptr;
            uint32_t total = 0;
            const uint32_t clamp = table_clamp(ne);
            if (!need_scan) {
                en = tabs.entries + a.slot;
                tab = tabs.table + (size_t)en->id * tabs.pitch + g.sbase;
                total = tabs.total[(size_t)en->id * tabs.n_groups + grp];
                // distribute-evenly: no hosting node at all -> no executor can be placed (distribute_evenly.go:72);
                // 1..k hosting nodes: several rounds or an exact per-candidate test -> the scan decides
                if (ALGO == 1 && k != 0 && total != 0 && total < k + 1) need_scan = true;
            }
            if (!need_scan && !(k != 0 && (ALGO == 0 ? total < k : total == 0))) {   // not even without a driver (pack_tightly.go:62, distribute_evenly.go:72)
                const bool drv_gpu = d_gpu != 0 || (snap_flags & kSnapGpuNegative);
                const bool cap_gpu = drv_gpu || (en->flags & 1u);
                const longlong2* gpair = s.pair + g.sbase;
                const int64_t* ggpu = s.gpu + g.sbase;
                // ---- driver loop (binpack.go:67-85) from the shape's first fitting candidate ---------------------------
                int32_t j = a.did >= 0 ? tabs.firstfit[(size_t)a.did * tabs.n_groups + grp] : 0;
                int32_t dslot = -1;
                uint32_t cd = 0, c0d = 0, sd = 0;
                for (; j < nd; ++j) {
                    ++drivers;
                    const int32_t ls = s.drv_slot[g.dbase + j];
                    const longlong2 v = __ldg(gpair + ls);
                    const int64_t gv = (drv_gpu || cap_gpu) ? __ldg(ggpu + ls) : 0;
                    if ((d_cpu > v.x) || (d_mem > v.y) || (drv_gpu && d_gpu > gv)) continue;
                    uint32_t my_c0 = 0, my_cd = 0, sp = 0;
                    if (ls < ne && k != 0) {
                        sp = tab[ls];
                        my_c0 = tab_at(tab, ls + 1, ne, total) - sp;
                        probes += 2;
                        if (my_c0 != 0) {        // what the node can still take once the driver sits on it
                            uint32_t c = min(cap_dim(v.x - d_cpu, en->div[0], clamp), cap_dim(v.y - d_mem, en->div[1], clamp));
                            if (cap_gpu) c = min(c, cap_dim(gv - d_gpu, en->div[2], clamp));
                            if (ALGO == 1) c = c != 0 ? 1u : 0u;
                            my_cd = c;
                        }
                        if (ALGO == 0 && total - (my_c0 - my_cd) < k) continue;       // the executors do not fit with this driver
                        // distribute-evenly: >= k+1 hosting nodes, the driver removes at most its own
                    }
                    dslot = ls; cd = my_cd; c0d = my_c0; sd = sp;
                    break;
                }
                if (dslot >= 0) {
                    result = s.slot_node[g.sbase + dslot];
                    // ---- emission by index shift: the driver's node takes cd instead of c0 executors, so every executor
                    // after its run comes delta = c0 - cd places later in the driver-free placement P:
                    //   out[t] = P[t < S(d) + cd ? t : t + delta]      (delta = 0 on a driver-only node: c0 = cd = 0)
                    // The warp writes these after the branch, coalesced; larger indices walk the table below.
                    const uint32_t delta = c0d - cd;
                    if (k != 0 && (uint64_t)k - 1u + delta < (uint64_t)kPlaceLen) {
                        sh_k = k; sh_delta = delta;
                        sh_cut = min(sd + cd, (uint32_t)kPlaceLen);     // S(d) + cd <= total; >= kPlaceLen: no shift below k
                        sh_dst = off;
                        sh_src = ((int64_t)en->id * tabs.n_groups + grp) * kPlaceLen;
                        probes += k;                            // one P word per executor
                    } else if (k != 0) {
                        // ---- emission: walk the prefix table from the first hosting node ---------------------------------
                        OUT* out = executor_nodes + off;
                        const int32_t* slot_node = s.slot_node + g.sbase;
                        const int32_t dpos = (dslot < ne) ? dslot : 0x7fffffff;
                        int32_t pos = tabs.first_host[(size_t)en->id * tabs.n_groups + grp];    // first node with room for the shape
                        ++probes;
                        uint32_t prev = 0, placed = 0;
                        uint32_t nxt = tab_at(tab, pos + 1, ne, total);
                        ++probes;
                        while (placed < k && pos < ne) {
                            // S(pos + 2) is requested before S(pos + 1) is consumed: the walk's dependent-load chain is
                            // what bounds this phase (one thread per application), so the next word is always in flight
                            const uint32_t nxt2 = tab_at(tab, pos + 2, ne, total);
                            ++probes;
                            uint32_t c = nxt - prev;
                            if (pos == dpos) c = cd;
                            if (c == 0) {                               // zero-capacity run (or the driver ate its node): jump
                                if (nxt >= total) break;                // cannot happen for a feasible placement
                                pos = tab_next_above(tab, pos + 1, ne, total, nxt, probes) - 1;
                                prev = nxt;
                                nxt = tab_at(tab, pos + 1, ne, total);
                                ++probes;
                                continue;
                            }
                            const uint32_t take = c < k - placed ? c : k - placed;
                            const OUT node = (OUT)__ldg(slot_node + pos);
                            for (uint32_t t = 0; t < take; ++t) out[placed + t] = node;
                            placed += take;
                            prev = nxt;
                            nxt = nxt2;
                            ++pos;
                        }
                    }
                }
            }
            if (need_scan) {
                // ---- prepared record for the scan kernel ------------------------------------------------------------------
                const int32_t at = atomicAdd(&tabs.hdr->n_listed, 1);
                PrepApp p;
                int b2 = 0; uint64_t lmax = 0; bool fast = true;
                const int64_t e_gpu = cols.load(5, i);
                const int64_t dd[3] = {d_cpu, d_mem, d_gpu}, ee[3] = {cols.load(3, i), cols.load(4, i), e_gpu};
#pragma unroll
                for (int t = 0; t < 3; ++t) {
                    uint64_t l;
                    p.drv[t] = dd[t];
                    p.div[t] = prep_dim(dd[t], ee[t], t, s.meta->max_avail[t], b2, l, fast);
                    if (l > lmax) lmax = l;
                }
                p.out_off = off; p.count = kk; p.group = grp;
                p.lmax = (int32_t)(lmax < (uint64_t)k ? lmax : (uint64_t)k);
                const bool f32 = prep_fast32(fast, p.div[0], p.div[1], s.meta);
                p.flags = ((d_gpu != 0 || e_gpu != 0) ? kAppUsesGpu : 0u) | (fast ? kAppFast : 0u) | (f32 ? kAppFast32 : 0u);
                const uint4* src = reinterpret_cast<const uint4*>(&p);
                uint4* dst = reinterpret_cast<uint4*>(prep + at);
#pragma unroll
                for (int t = 0; t < (int)(sizeof(PrepApp) / sizeof(uint4)); ++t) dst[t] = src[t];
                listed[at] = i;
            } else {
                driver_node[i] = result;
            }
        }
    }
    // ---- coalesced emission of the index-shift lanes: the warp's executor indices are concatenated in lane order, and
    // every 32-index chunk is written by the whole warp (owner lane of index e: binary search over the inclusive scan).
    // kEmitBatch chunks per round: their owner searches are independent shuffle chains, and all their P loads are issued
    // before the first store, so a round costs one load round trip instead of one per chunk.
    {
        constexpr int kEmitBatch = 4;
        const uint32_t incl = warp_incl_scan(sh_k, lane);
        const uint32_t n_out = __shfl_sync(kFull, incl, 31);
        const uint32_t excl = incl - sh_k;
        const int64_t dst = sh_dst - (int64_t)excl, src = sh_src - (int64_t)excl;     // index e of the concatenation
        const uint32_t cut = excl + sh_cut;
        for (uint32_t e0 = 0; e0 < n_out; e0 += 32 * kEmitBatch) {
            int owner[kEmitBatch];                      // number of lanes whose indices all lie before e
            int32_t node[kEmitBatch];
#pragma unroll
            for (int b = 0; b < kEmitBatch; ++b) {
                const uint32_t e = e0 + 32u * b + (uint32_t)lane;
                int o = 0;
#pragma unroll
                for (int step = 16; step >= 1; step >>= 1)
                    if (__shfl_sync(kFull, incl, o + step - 1) <= e) o += step;
                const int64_t o_src = __shfl_sync(kFull, src, o);
                const uint32_t o_cut = __shfl_sync(kFull, cut, o), o_delta = __shfl_sync(kFull, sh_delta, o);
                owner[b] = o;
                node[b] = e < n_out ? tabs.place[o_src + e + (e < o_cut ? 0u : o_delta)] : 0;
            }
#pragma unroll
            for (int b = 0; b < kEmitBatch; ++b) {
                const uint32_t e = e0 + 32u * b + (uint32_t)lane;
                const int64_t o_dst = __shfl_sync(kFull, dst, owner[b]);
                if (e < n_out) executor_nodes[o_dst + e] = (OUT)node[b];
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// the one launch: classify -> tables -> decide
// ---------------------------------------------------------------------------------------------------------------
// A persistent grid (sized by the occupancy query) works off one sequence of work items.  Every CTA claims the next
// ticket with atomicAdd on hdr->ticket, runs the item, and claims again:
//   tickets [0, n_cls)                  classify tiles of kTabThreads applications (n_cls = 0 when neither the tables nor
//                                       the offsets are needed);
//   [n_cls, n_cls + n_tab)              table items, known once every classify tile is done: per executor shape present
//                                       and group, its segments in order (seg_pre), then per (driver shape, group) one
//                                       first-fit item;
//   any later ticket                    the CTA turns to the decide phase: warp w of CTA b first takes 32-application chunk
//                                       b * 8 + w, with no claim; chunks past the grid's warp count are claimed one per
//                                       warp from hdr->dec_next until none is left (the cost of a decision varies with
//                                       its walk; warp-sized claims keep the SMs evenly loaded), then the CTA leaves.
// Forward progress.  An item waits only for items with smaller tickets: a classify tile for the tiles before it (offset
// look-back), a table item for every classify tile (hdr->cls_done) and for the earlier segments of its (shape, group)
// (look-back), the decide phase for every table item (hdr->tab_done).  A ticket is claimed by a CTA that is running, and a
// CTA claims its next ticket only after finishing the last one.  So by induction over the tickets, every claimed item
// completes, whatever number of CTAs happens to be co-resident (other work on the GPU, the other pipeline lanes).
// A decide chunk waits on nothing once the tables are done, so giving each warp a fixed first chunk by blockIdx is safe:
// every CTA of the grid runs eventually and reaches the decide phase.  Tickets stay dynamic: CTAs are not dispatched
// in index order, and a fixed ticket could make a running CTA wait for one that has not started.
// The ticket, the phase counters and every look-back word start from zero: the previous call's gp_pack_listed left them so.
// The item with ticket 0 is always a classify tile (one tile with nothing to classify when neither the tables nor the
// offsets are needed).  It zeroes hdr->n_listed and, with status_zero != NULL, the call's status block (kStatusWords
// words: error bits, statistics, claim counters) instead of a memset before the launch.  It finishes before cls_done can
// count every tile, and every CTA waits for that count before it appends to the list, writes the error word or adds to
// the statistics, so no write of the call is lost to the zeroing.
// Early start (programmatic dependent launch).  The host may launch this kernel while the slot layout that precedes it
// on the stream (gp_build_slots_drv) is still running (launch_tables, early_start).  So the classify tiles read nothing
// of the snapshot: they read the application columns and offsets, and write app_slot, the hash entries, the look-back
// words, the ticket, n_listed and the status block, none of which the layout kernels touch.  Every CTA runs pdl_wait()
// right after its cls_done wait, before its first read of seg_pre, s.groups or anything else of the snapshot; every
// table item and every decide chunk comes after it.  The host allows the early start only when the application columns
// were ready before the layout was enqueued (gangpack.h, GP_CFG_ASYNC_SNAPSHOT).  Forward progress is as above: this
// kernel starts only once every CTA of gp_build_slots_drv has run pdl_trigger(), so every CTA it waits for is already
// resident and finishes whatever this grid occupies.  Each CTA runs pdl_trigger() as it leaves, for gp_pack_listed.
template <int ALGO, class OUT>
__global__ void __launch_bounds__(kTabThreads) gp_decide_tables(Snapshot s, AppColumns cols, ShapeTables tabs, int64_t off_base,
                                                                int64_t* off_out /* or NULL */, int32_t* app_slot, int32_t n_apps,
                                                                int64_t out_cap, int32_t* __restrict__ driver_node,
                                                                OUT* __restrict__ executor_nodes, PrepApp* __restrict__ prep,
                                                                int32_t* __restrict__ listed, unsigned long long* __restrict__ stats,
                                                                int* __restrict__ err, volatile int* __restrict__ err_host, int force_scan,
                                                                unsigned int* __restrict__ status_zero) {
    __shared__ OneScratch sh;
    ShapeHeader* hdr = tabs.hdr;
    const int32_t n_tiles = (n_apps + kTabThreads - 1) / kTabThreads;
    const int32_t n_cls = (!force_scan || off_out) ? n_tiles : 1;
    int32_t n_es = 0, n_tab = -1, total_segs = 0;         // n_tab < 0: classify not yet seen complete by this CTA
    unsigned long long probes = 0, drivers = 0;
    GP_TL(uint32_t tl_n = 0; unsigned long long tl_t0 = 0;)
    for (;;) {
        if (threadIdx.x == 0) sh.ticket = atomicAdd(&hdr->ticket, 1u);
        GP_TL(if (threadIdx.x == 0) tl_t0 = tl_now();)
        __syncthreads();
        const int32_t t = (int32_t)sh.ticket;
        if (t < n_cls) {
            if (t == 0) {
                if (threadIdx.x == 0) hdr->n_listed = 0;
                if (status_zero && threadIdx.x < kStatusWords) status_zero[threadIdx.x] = 0u;
            }
            if (off_out) classify_offsets(sh, t, n_apps, cols, tabs, off_base, off_out);
            if (!force_scan) gp_classify_apps(t, n_apps, cols, tabs, app_slot);
            signal_done(&hdr->cls_done);
            GP_TL(if (threadIdx.x == 0) tl_rec(tl_n, kTlCls, (uint32_t)t, tl_t0);)
            continue;
        }
        if (n_tab < 0) {
            if (threadIdx.x == 0) {
                GP_TL(const unsigned long long w0 = tl_now();)
                wait_count(&hdr->cls_done, (uint32_t)n_cls);
                GP_TL(tl_rec(tl_n, kTlClsWait, 0u, w0);)
            }
            __syncthreads();
            pdl_wait();                 // the slot layout has ended: everything below may read the snapshot
            n_tab = 0;
            if (!force_scan) {
                n_es = min(hdr->n_shapes, kMaxShapes);
                total_segs = tabs.seg_pre[s.n_groups];
                n_tab = n_es * total_segs + min(hdr->n_dshapes, kMaxShapes) * s.n_groups;
            }
        }
        int32_t r = t - n_cls;
        if (r < n_tab) {
            if (r < n_es * total_segs) {
                const int id = r / total_segs;
                const int32_t gs = r - id * total_segs;
                int32_t lo = 0, hi = s.n_groups - 1;          // the group whose segments [seg_pre[g], seg_pre[g+1]) hold gs
                while (lo < hi) {
                    const int32_t mid = (lo + hi + 1) >> 1;
                    if (tabs.seg_pre[mid] <= gs) lo = mid; else hi = mid - 1;
                }
                const int32_t s0 = tabs.seg_pre[lo];
                gp_build_shape_tables<ALGO>(sh, s, tabs, id, lo, gs - s0, tabs.seg_pre[lo + 1] - s0, tabs.seg_status + r);
            } else {
                const int32_t rd = r - n_es * total_segs;
                driver_firstfit_block(s, tabs, rd / s.n_groups, rd % s.n_groups);
            }
            signal_done(&hdr->tab_done);
            GP_TL(if (threadIdx.x == 0) tl_rec(tl_n, r < n_es * total_segs ? kTlSeg : kTlFirstFit, (uint32_t)r, tl_t0);)
            continue;
        }
        // The warp's first chunk is fixed, and everything decide_load reads was written before cls_done (which this CTA
        // has seen): its loads are in flight while thread 0 waits for the tables.
        const int lane = threadIdx.x & 31;
        GP_TL(unsigned long long tl_w0 = 0; uint32_t tl_chunks = 0;)
        const uint32_t n_chunks = (uint32_t)(n_apps + 31) / 32u, n_warps = gridDim.x * (kTabThreads / 32u);
        uint32_t c = blockIdx.x * (kTabThreads / 32u) + (threadIdx.x >> 5);
        AppIn a = decide_load((int32_t)c * 32 + lane, s, cols, tabs, app_slot, n_apps, out_cap, force_scan);
        if (threadIdx.x == 0) {
            GP_TL(const unsigned long long w0 = tl_now();)
            wait_count(&hdr->tab_done, (uint32_t)n_tab);
            GP_TL(tl_rec(tl_n, kTlTabWait, 0u, w0);)
        }
        __syncthreads();
        while (c < n_chunks) {
            GP_TL(if (tl_chunks++ == 0) tl_w0 = tl_now();)
            decide_app<ALGO, OUT>((int32_t)c * 32 + lane, a, s, cols, tabs, driver_node, executor_nodes, prep, listed, err, err_host,
                                  probes, drivers);
            // the chunks past the grid's warps: claimed one at a time (their cost varies with the walks), and only while
            // the counter says some are left
            c = n_chunks;
            if (n_warps < n_chunks) {
                if (lane == 0 && n_warps + ld_relaxed_u32(&hdr->dec_next) < n_chunks) c = n_warps + atomicAdd(&hdr->dec_next, 1u);
                c = __shfl_sync(kFull, c, 0);
                if (c < n_chunks) a = decide_load((int32_t)c * 32 + lane, s, cols, tabs, app_slot, n_apps, out_cap, force_scan);
            }
        }
        GP_TL(if (lane == 0 && blockIdx.x < kTlCtas) {
            const uint32_t gw = blockIdx.x * (kTabThreads / 32) + (threadIdx.x >> 5);
            g_tl.warp[gw][0] = tl_w0; g_tl.warp[gw][1] = tl_chunks ? tl_now() : 0ull; g_tl.warp_chunks[gw] = tl_chunks;
        })
        GP_TL(if (threadIdx.x == 0) {
            if (blockIdx.x < kTlCtas) g_tl.n[blockIdx.x] = tl_n;
            if (blockIdx.x == 0) { g_tl.grid = gridDim.x; g_tl.n_cls = (uint32_t)n_cls; g_tl.n_tab = (uint32_t)n_tab; g_tl.n_chunks = (uint32_t)(n_apps + 31) / 32u; }
        })
        break;
    }
    // statistics: one atomic per warp
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) { probes += __shfl_xor_sync(kFull, probes, d); drivers += __shfl_xor_sync(kFull, drivers, d); }
    if ((threadIdx.x & 31) == 0 && (probes | drivers)) { atomicAdd(stats + 0, probes); atomicAdd(stats + 1, drivers); }
    pdl_trigger();
}

// ---------------------------------------------------------------------------------------------------------------
// the node-order scan for the listed applications: one warp per application (gangpack_kernels.cuh)
// ---------------------------------------------------------------------------------------------------------------
constexpr int kPackTabThreads = 256;
#ifndef GP_TAB_MIN_BLOCKS
#define GP_TAB_MIN_BLOCKS 4
#endif
// It is the last kernel of every call on its table set, so it also leaves the set clean for the next call: its CTAs zero
// the counters, the hash keys and the n_cls_words / n_seg_words look-back words the call used (a claimer writes every
// other field of a hash entry).  It is launched as gp_decide_tables' dependent and may start while that kernel's last CTAs
// are leaving; every CTA waits for gp_decide_tables to finish (pdl_wait) before it reads n_listed or zeroes anything.  No
// CTA sizes its share from a header word, and n_listed, which they read, is left to the next call.
template <int ALGO, class OUT>
__global__ void __launch_bounds__(kPackTabThreads, GP_TAB_MIN_BLOCKS) gp_pack_listed(Snapshot s, ShapeTables tabs, int32_t n_cls_words,
                                                                                     int32_t n_seg_words,
                                                                                     const PrepApp* __restrict__ prep,
                                                                                     const int32_t* __restrict__ listed,
                                                                                     int32_t* __restrict__ driver_node,
                                                                                     OUT* __restrict__ executor_nodes,
                                                                                     int2* __restrict__ scratch,
                                                                                     unsigned long long* __restrict__ stats,
                                                                                     unsigned int* __restrict__ next_app) {
    __shared__ uint16_t cap_cache[kPackTabThreads / 32][kCapCache];
    ShapeHeader* hdr = tabs.hdr;
    pdl_wait();
    const int n = hdr->n_listed;
    {
        const int32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
        if (tid == 0) {
            hdr->n_shapes = 0; hdr->n_dshapes = 0;
            hdr->ticket = 0; hdr->cls_done = 0; hdr->tab_done = 0; hdr->dec_next = 0;
        }
        for (int32_t k = tid; k < kShapeSlots; k += nth) { tabs.entries[k].key = 0ull; tabs.dentries[k].key = 0ull; }
        for (int32_t k = tid; k < n_cls_words; k += nth) tabs.cls_status[k] = 0ull;
        for (int32_t k = tid; k < n_seg_words; k += nth) tabs.seg_status[k] = 0ull;
    }
    if (n != 0) {
        const int lane = threadIdx.x & 31;
        uint16_t* wcache = cap_cache[threadIdx.x >> 5];
        WarpStats st{0, 0};
        const int snap_flags = s.meta->flags;
        const GroupDesc g0 = s.groups[0];
        unsigned int i = 0, n1 = 0;
        if (lane == 0) { i = atomicAdd(next_app, 1u); n1 = atomicAdd(next_app, 1u); }
        i = __shfl_sync(kFull, i, 0);
        n1 = __shfl_sync(kFull, n1, 0);
        unsigned long long apps_done = 0;
        while (i < (unsigned int)n) {
            unsigned int n2 = 0;
            if (lane == 0) n2 = atomicAdd(next_app, 1u);
            if (lane == 0 && n1 < (unsigned int)n) asm volatile("prefetch.global.L1 [%0];" ::"l"(prep + n1));
            const PrepApp* pa = prep + i;
            const int32_t d = pack_app<ALGO, OUT>(s, pa, executor_nodes, scratch, wcache, st, lane, snap_flags, g0);
            if (lane == 0) driver_node[listed[i]] = d;
            ++apps_done;
            i = n1;
            n1 = __shfl_sync(kFull, n2, 0);
        }
        if (lane == 0) {
            atomicAdd(stats + 0, st.nodes);
            atomicAdd(stats + 1, st.drivers);
            atomicAdd(stats + 2, apps_done);
            atomicAdd(stats + 3, st.nodes);
        }
    }
}

}  // namespace gp

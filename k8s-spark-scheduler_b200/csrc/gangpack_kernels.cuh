// gangpack_kernels.cuh -- sm_90a device code of the gang-placement hot path.
//
// What is computed (reference, all under /root/reference; LIB = vendor/github.com/palantir/
// k8s-spark-scheduler-lib/pkg):
//   SparkBinPack driver loop            LIB/binpack/binpack.go:60-87
//   tightlyPackExecutors                LIB/binpack/pack_tightly.go:34-63
//   distributeExecutorsEvenly           LIB/binpack/distribute_evenly.go:34-73
//   Resources.GreaterThan / Add / Sub   LIB/resources/resources.go:239-241, 202-213
//   fitEarlierDrivers + sparkResourceUsage + SubtractUsageIfExists
//                                       internal/extender/resource.go:224-262,
//                                       internal/extender/sparkpods.go:139-146,
//                                       LIB/resources/resources.go:129-135
//
// How (GPU-first, not a translation): the reference re-runs the executor loop for every driver
// candidate over string-keyed maps.  Here a node's executor capacity is a closed form
// (the reference's own LIB/capacity/capacity.go:36-75):
//     cap_dim(n|r) = 0 if r > avail ; INF if exe == 0 ; floor((avail - r) / exe)
//     cap(n|r)     = min over cpu, mem, gpu
// so one WARP owns one pending application, lanes own consecutive nodes of the executor
// priority order (coalesced 128-bit (cpu,mem) loads), a warp reduction/prefix scan counts the
// executors that fit, lanes trial-place the driver on 32 candidates at a time and
// __ballot_sync picks the first feasible one, and a second pass emits ExecutorNodes.
// Division by the (warp-uniform) executor request is a multiply-high by a per-app magic
// number computed once by gp_prep_apps (exact, see cap_dim()).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace gp {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr int32_t kMaxCount = 1 << 24;            // exe_count limit (keeps 32-lane int32 sums exact)
constexpr int32_t kMaxCountFifo = 1 << 20;        // FIFO modes: 1024 threads x min(cap, k) must stay below 2^32
constexpr int64_t kMaxQuantity = (int64_t)1 << 61; // |quantity| limit of the exact-int64 domain

// error bits raised by device-side validation (read back by the host API)
enum : int {
    kErrNegativeRequest = 1,   // driver/executor request < 0 or exe_count < 0
    kErrUnrepresentable = 2,   // |quantity| >= 2^61 or exe_count > 2^24
    kErrBadGroup = 4,          // app group outside [0, n_groups)
    kErrBadOffsets = 8,        // exec_out_off inconsistent with exe_count / capacity
};

// snapshot flags (device int) -- SnapMeta::flags
enum : int { kSnapGpuNegative = 1 };

// Per-snapshot facts the kernels need: flags + the largest availability per dimension (a node's
// availability only ever decreases afterwards, so the maxima stay upper bounds in FIFO modes).
struct SnapMeta {
    int flags;
    int pad;
    long long max_avail[3];   // cpu milli, mem bytes, gpu
    int shift32[2];           // compact view: pair32 = (max(cpu,0) >> shift32[0], max(mem,0) >> shift32[1]), both < 2^32
    int pad2[2];
};

// How to divide by one executor-request dimension.
enum : uint32_t { kDivInf = 0, kDivMagic = 1, kDivShift = 2, kDivSlow = 3 };

struct DimDiv {
    uint64_t magic;  // floor((2^64-1)/e') + 1 for e = e' << sh, e' < 2^32   (kDivMagic)
    int64_t e;       // the request itself
    uint32_t sh;     // trailing zero bits of e
    uint32_t kind;
};

// One pending application, prepared (128 B).
struct __align__(16) PrepApp {
    int64_t drv[3];      // driver cpu, mem, gpu
    DimDiv div[3];       // executor cpu, mem, gpu
    int64_t out_off;     // first ExecutorNodes slot of this app
    int32_t count;       // MinExecutorCount
    int32_t group;
    int32_t lmax;        // max executors the driver can displace on its own node (<= count)
    uint32_t flags;      // bit0: uses gpu dim, bit1: skip_if_no_fit, bit2: invalid, bit3: fast class, bit4: compact 32-bit view usable
};
enum : uint32_t { kAppUsesGpu = 1u, kAppSkipIfNoFit = 2u, kAppInvalid = 4u, kAppFast = 8u, kAppFast32 = 16u };
static_assert(sizeof(PrepApp) == 128, "PrepApp layout");

// Smallest requests over the batch's applications of one instance group (gp_prep_apps, atomicMin).
// A node with avail < min request in some dimension can host nothing for ANY application of the batch,
// and availability only decreases in the FIFO loop -> such nodes can be skipped for good.
struct GroupMin {
    long long exe[3];   // min executor cpu, mem, gpu (0 = some app asks nothing in that dimension)
    long long drv[3];   // min driver   cpu, mem, gpu
};

struct GroupDesc {
    int32_t sbase;   // first slot of the group
    int32_t ne;      // executor-order length: slots [sbase, sbase+ne) in priority order
    int32_t dbase;   // first entry in drv_slot
    int32_t nd;      // driver-order length
};

// Independent-mode capacity tables (gangpack_tables.cuh) are built in segments of kTabSeg executor-order positions.  The
// slot layout counts each group's segments once per snapshot (gp_build_slots_drv), so a pack call need not.
constexpr int kTabThreads = 256;      // every phase of gp_decide_tables; also the applications per classify tile
constexpr int kTabPerThread = 4;
constexpr int kTabSeg = kTabThreads * kTabPerThread;      // nodes per table segment

// Programmatic dependent launch (sm_90).  A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may
// start once every CTA of the kernel before it on the stream has run pdl_trigger() or exited; its pdl_wait() returns once
// that kernel has completed and its writes are visible.  Without the attribute pdl_wait() returns at once.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Device snapshot: "slots" = per group the executor order followed by one spare slot per driver
// candidate (used only when that candidate is not an executor candidate).
struct Snapshot {
    longlong2* pair;       // [n_slots] (avail cpu milli, avail mem bytes)
    const uint2* pair32;   // [n_slots] compact read-only view of `pair` (see SnapMeta::shift32); independent mode only
    int64_t* gpu;          // [n_slots]
    int32_t* slot_node;    // [n_slots] caller's node index, -1 = unused spare
    const int32_t* drv_slot; // [n_drv] group-local slot of each driver candidate
    const GroupDesc* groups;
    const SnapMeta* meta;
    const GroupMin* gmins;   // FIFO modes only
    int32_t n_groups;
    int32_t n_slots;
};

// ---- raw application columns in either wire width --------------------------------------------------------------
// 64-bit layout: exact int64 quantities (gp_apps).  32-bit layout (gp_apps_wire.quantity_bits == 32): int32 millicores /
// int32 (bytes >> mem_shift) / int32 gpu units -- 28 bytes per application instead of 60.
struct AppColumns {
    const void* q[6];                 // drv cpu, drv mem, drv gpu, exe cpu, exe mem, exe gpu (gpu columns may be NULL = 0)
    const int32_t* count;
    const int32_t* group;             // or NULL (= 0)
    const int64_t* off;               // [n+1] ExecutorNodes offsets (the caller's, or the ones K1 derived)
    int32_t bits;                     // 64 or 32
    int32_t mem_shift;                // 32-bit layout only
    __device__ __forceinline__ int64_t load(int c, int32_t i) const {
        const void* p = q[c];
        if (!p) return 0;
        if (bits == 64) return static_cast<const int64_t*>(p)[i];
        const int64_t v = static_cast<const int32_t*>(p)[i];
        return (c == 1 || c == 4) ? (v < 0 ? v : (v << mem_shift)) : v;     // negative stays negative -> validation error
    }
};

// words of a pack call's status block (the host's DevStatus), which gp_decide_tables can zero in place of a memset
constexpr int kStatusWords = 32;

// fingerprint of a (cpu, mem, gpu) request, never 0: the shape hashes of gp_decide_tables and gp_cc_intern
__host__ __device__ __forceinline__ unsigned long long shape_fingerprint(int64_t a, int64_t b, int64_t c) {
    unsigned long long z = (unsigned long long)a * 0x9E3779B97F4A7C15ull;
    z ^= ((unsigned long long)b + 0xBF58476D1CE4E5B9ull) * 0x94D049BB133111EBull;
    z ^= ((unsigned long long)c + 0x2545F4914F6CDD1Dull) * 0xD6E8FEB86659FD93ull;
    z ^= z >> 29; z *= 0xBF58476D1CE4E5B9ull; z ^= z >> 32;
    return z ? z : 1ull;
}

// ---------------------------------------------------------------------------------------------
// capacity arithmetic
// ---------------------------------------------------------------------------------------------
// Executors of request e that fit into `a` free units:  a < 0 -> 0 (reserved > avail in this
// dimension, resources.go:239); e == 0 -> unlimited; else floor(a / e).
// Exact division by the warp-uniform request: e = e' << sh, a >= 0  =>  floor(a/e) = floor((a >> sh)/e');
// for xs = a >> sh < 2^32 and e' < 2^32, floor(xs/e') = mulhi64(magic, xs) with
// magic = floor((2^64-1)/e') + 1 (Lemire, Kaser, Kurz 2019, N = 32).

// static: not inline, and several translation units of the library include this header
static __device__ __noinline__ uint64_t udiv64(uint64_t a, uint64_t b) { return a / b; }

// ---- general class: any int64 request ----------------------------------------------------------
__device__ __forceinline__ uint32_t cap_dim(int64_t a, const DimDiv& p, uint32_t k) {
    if (a < 0) return 0;
    if (p.kind == kDivInf) return k;
    uint64_t xs = (uint64_t)a >> p.sh;
    uint64_t q;
    if (p.kind == kDivShift) q = xs;
    else if (p.kind == kDivMagic && (xs >> 32) == 0) q = __umul64hi(p.magic, xs);
    else q = udiv64((uint64_t)a, (uint64_t)p.e);
    return q < (uint64_t)k ? (uint32_t)q : k;
}

// ---- fast class: every dimension has (max_avail >> sh) < 2^32 and e' < 2^32 (decided per app by
// gp_prep_apps from SnapMeta::max_avail) -> branch-free 32-bit arithmetic ---------------------------
struct FastDim {
    uint32_t m_lo, m_hi;   // magic
    uint32_t sh;           // 0..63
    uint32_t mode;         // kDivMagic / kDivShift / kDivInf
};
__device__ __forceinline__ FastDim fast_dim(const DimDiv& d) {
    FastDim f;
    f.m_lo = (uint32_t)d.magic; f.m_hi = (uint32_t)(d.magic >> 32); f.sh = d.sh; f.mode = d.kind;
    return f;
}
__device__ __forceinline__ uint32_t fast_q(int64_t a, const FastDim& p) {
    const uint32_t lo = (uint32_t)a, hi = (uint32_t)((uint64_t)a >> 32);
    const bool big = p.sh >= 32;
    const uint32_t xs = __funnelshift_r(big ? hi : lo, big ? 0u : hi, p.sh & 31);   // (a >> sh), known < 2^32
    uint32_t q = (uint32_t)(((uint64_t)p.m_hi * xs + __umulhi(p.m_lo, xs)) >> 32);  // mulhi64(magic, xs)
    q = p.mode == kDivShift ? xs : q;
    q = p.mode == kDivInf ? 0xFFFFFFFFu : q;
    return (int32_t)hi < 0 ? 0u : q;
}

// cpu / mem dimensions of the fast class are always kDivMagic (a power-of-two request 2^sh is prepared as
// "divide (a >> (sh-1)) by 2", magic 2^63): no mode selects in the hot loop.
__device__ __forceinline__ uint32_t fast_q_magic(int64_t a, const FastDim& p) {
    const uint32_t lo = (uint32_t)a, hi = (uint32_t)((uint64_t)a >> 32);
    const bool big = p.sh >= 32;
    const uint32_t xs = __funnelshift_r(big ? hi : lo, big ? 0u : hi, p.sh & 31);
    const uint32_t q = (uint32_t)(((uint64_t)p.m_hi * xs + __umulhi(p.m_lo, xs)) >> 32);
    return (int32_t)hi < 0 ? 0u : q;
}

template <bool MUTABLE>
__device__ __forceinline__ longlong2 load_pair(const longlong2* p) {
    if (MUTABLE) {
        longlong2 v;
        asm volatile("ld.global.v2.s64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
        return v;
    } else {
        return __ldg(p);
    }
}
template <bool MUTABLE>
__device__ __forceinline__ int64_t load_gpu(const int64_t* p) {
    if (MUTABLE) {
        int64_t v;
        asm volatile("ld.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
        return v;
    } else {
        return __ldg(p);
    }
}

__device__ __forceinline__ uint32_t warp_sum(uint32_t v) { return __reduce_add_sync(kFull, v); }

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < kWarp; d <<= 1) {
        uint32_t t = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += t;
    }
    return v;
}
__device__ __forceinline__ uint32_t umin3(uint32_t a, uint32_t b, uint32_t c) { return min(min(a, b), c); }

// ---------------------------------------------------------------------------------------------
// per-application capacity calculators (registers of one warp)
// ---------------------------------------------------------------------------------------------
template <bool FAST> struct Caps;

template <> struct Caps<true> {
    FastDim cpu, mem, gpu;
    int64_t d_cpu, d_mem, d_gpu;
    int64_t e_cpu, e_mem, e_gpu;
    uint32_t k;
    bool use_gpu;
    __device__ __forceinline__ void init(const PrepApp* pa, bool ug) {
        d_cpu = pa->drv[0]; d_mem = pa->drv[1]; d_gpu = pa->drv[2];
        cpu = fast_dim(pa->div[0]); mem = fast_dim(pa->div[1]); gpu = fast_dim(pa->div[2]);
        e_cpu = pa->div[0].e; e_mem = pa->div[1].e; e_gpu = pa->div[2].e;
        k = (uint32_t)pa->count; use_gpu = ug;
    }
    // Compact view: both availabilities pre-shifted to 32 bits (negative -> 0, which also yields capacity 0 because
    // the requests of this class are > 0).  a >> sh == (a >> S) >> (sh - S) for sh >= S, so the quotient is the same.
    uint32_t sh32_cpu, sh32_mem;    // sh - S per dimension (kAppFast32 only)
    __device__ __forceinline__ void init32(const SnapMeta* meta) {
        sh32_cpu = cpu.sh - (uint32_t)meta->shift32[0];
        sh32_mem = mem.sh - (uint32_t)meta->shift32[1];
    }
    __device__ __forceinline__ uint32_t cap32(uint2 v) const {
        const uint32_t xc = v.x >> sh32_cpu, xm = v.y >> sh32_mem;
        const uint32_t qc = (uint32_t)(((uint64_t)cpu.m_hi * xc + __umulhi(cpu.m_lo, xc)) >> 32);
        const uint32_t qm = (uint32_t)(((uint64_t)mem.m_hi * xm + __umulhi(mem.m_lo, xm)) >> 32);
        return umin3(qc, qm, k);
    }
    // capacity from already-loaded availability, reservation r, clamped to k
    __device__ __forceinline__ uint32_t cap_pair(longlong2 v, int64_t r_cpu, int64_t r_mem) const {
        return umin3(fast_q_magic(v.x - r_cpu, cpu), fast_q_magic(v.y - r_mem, mem), k);
    }
    template <bool MUT>
    __device__ __forceinline__ uint32_t cap(const Snapshot& s, int32_t slot, int64_t r_cpu, int64_t r_mem, int64_t r_gpu, bool ug) const {
        uint32_t c = cap_pair(load_pair<MUT>(s.pair + slot), r_cpu, r_mem);
        if (ug) c = min(c, fast_q(load_gpu<MUT>(s.gpu + slot) - r_gpu, gpu));
        return c;
    }
    template <bool MUT>
    __device__ __forceinline__ uint32_t cap0(const Snapshot& s, int32_t slot, bool ug) const { return cap<MUT>(s, slot, 0, 0, 0, ug); }
};

template <> struct Caps<false> {
    DimDiv cpu, mem, gpu;
    int64_t d_cpu, d_mem, d_gpu;
    int64_t e_cpu, e_mem, e_gpu;
    uint32_t k;
    bool use_gpu;
    __device__ __forceinline__ void init(const PrepApp* pa, bool ug) {
        d_cpu = pa->drv[0]; d_mem = pa->drv[1]; d_gpu = pa->drv[2];
        cpu = pa->div[0]; mem = pa->div[1]; gpu = pa->div[2];
        e_cpu = cpu.e; e_mem = mem.e; e_gpu = gpu.e;
        k = (uint32_t)pa->count; use_gpu = ug;
    }
    template <bool MUT>
    __device__ __forceinline__ uint32_t cap(const Snapshot& s, int32_t slot, int64_t r_cpu, int64_t r_mem, int64_t r_gpu, bool ug) const {
        longlong2 v = load_pair<MUT>(s.pair + slot);
        uint32_t c = min(cap_dim(v.x - r_cpu, cpu, k), cap_dim(v.y - r_mem, mem, k));
        if (ug) c = min(c, cap_dim(load_gpu<MUT>(s.gpu + slot) - r_gpu, gpu, k));
        return c;
    }
    template <bool MUT>
    __device__ __forceinline__ uint32_t cap0(const Snapshot& s, int32_t slot, bool ug) const { return cap<MUT>(s, slot, 0, 0, 0, ug); }
    __device__ __forceinline__ void init32(const SnapMeta*) {}
    __device__ __forceinline__ uint32_t cap32(uint2) const { return 0; }   // never instantiated with C32
};

// driverResources.GreaterThan(available) == false  (binpack.go:69)
template <bool MUT, class C>
__device__ __forceinline__ bool driver_fits(const Snapshot& s, int32_t slot, const C& a, bool ug) {
    longlong2 v = load_pair<MUT>(s.pair + slot);
    bool ok = !(a.d_cpu > v.x) && !(a.d_mem > v.y);
    if (ug) ok = ok && !(a.d_gpu > load_gpu<MUT>(s.gpu + slot));
    return ok;
}

// distribute-evenly, general rounds (distribute_evenly.go:49-70) over the complete candidate list
// (m <= k entries (position, cap) in priority order), executed by ONE warp:
// R* = min r with sum min(c, r) >= k; round r hands one executor to every node with c >= r until k are
// placed; ExecutorNodes is round-major.  charge1(local_slot) subtracts one executor (FIFO modes).
// Returns whether the driver's node received an executor.
template <int FIFO_MODE, class OUT, class ChargeFn>
__device__ __forceinline__ bool evenly_rounds(int2* __restrict__ list, uint32_t m, uint32_t k, int32_t dslot, uint32_t cd,
                                              OUT* __restrict__ out, const int32_t* __restrict__ slot_node, int lane,
                                              ChargeFn charge1) {
    bool driver_hosts_executor = false;
    for (uint32_t t = lane; t < m; t += kWarp) {   // patch the driver's own entry with cap(d|drv)
        int2 e = list[t];
        if (e.x == dslot) { e.y = (int)cd; list[t] = e; }
    }
    __syncwarp();
    uint32_t lo = 1, hi = k;   // f(k) >= k is known (feasible)
    while (lo < hi) {
        uint32_t mid = lo + (hi - lo) / 2;
        unsigned long long f = 0;
        for (uint32_t t0 = 0; t0 < m; t0 += kWarp) {
            uint32_t t = t0 + lane;
            uint32_t c = (t < m) ? (uint32_t)list[t].y : 0u;
            f += warp_sum(c < mid ? c : mid);
        }
        if (f >= k) hi = mid; else lo = mid + 1;
    }
    const uint32_t R = lo;
    uint32_t base = 0;
    for (uint32_t r = 1; r <= R && base < k; ++r) {
        for (uint32_t t0 = 0; t0 < m && base < k; t0 += kWarp) {
            uint32_t t = t0 + lane;
            int2 e = (t < m) ? list[t] : make_int2(0, 0);
            bool in = (t < m) && ((uint32_t)e.y >= r);
            unsigned has = __ballot_sync(kFull, in);
            uint32_t idx = base + __popc(has & ((1u << lane) - 1u));
            if (in && idx < k) {
                out[idx] = (OUT)slot_node[e.x];
                if (FIFO_MODE == 2 || (FIFO_MODE == 1 && r == 1)) charge1(e.x);
                if (FIFO_MODE != 0 && e.x == dslot) driver_hosts_executor = true;
            }
            base += __popc(has);
        }
    }
    return driver_hosts_executor;
}

struct WarpStats { unsigned long long nodes; unsigned long long drivers; };

constexpr int kCapCache = 1024;   // per-warp shared-memory cache of phase-1 capacities (uint16)

// Where pack_app_impl finds the nodes it scans (slot-mapping policy).
// GroupSlots: one instance group of the snapshot -- executor-order position i is slot g.sbase + i, driver candidate j has
//   the group-local slot drv_slot[g.dbase + j] (>= ne: its spare slot).
// GatherSlots: the undivided orders of az-aware-tightly-pack's fallback (gangpack_zonefifo.cuh), which run across instance
//   groups -- position i is slot exec_slot[i], driver candidate j is slot drv_slot[j] and executor-order position
//   drv_pos[j] (-1: not an executor candidate).  Every node has exactly one slot (node_slot), so a charge made through
//   either view is seen by both.
struct GroupSlots { static constexpr bool kGather = false; };
struct GatherSlots {
    static constexpr bool kGather = true;
    const int32_t* exec_slot;   // [ne]
    const int32_t* drv_slot;    // [nd]
    const int32_t* drv_pos;     // [nd]
    int32_t ne, nd;
};

constexpr int kZoneAzAware = 3;               // ALGO of az-aware-tightly-pack (0 and 2 are the single-AZ packers)

// One instance group of the zone FIFO loop (gp_pack_fifo_zones_cta, gangpack_zonefifo.cuh): CTA b runs the b-th
struct ZoneFifoGroup {
    int64_t row_base;                 // its scratch rows start at entry row_base of the row arrays
    int64_t row_pitch;                // >= max exe_count of its applications, a multiple of 4
    int32_t zone0, n_zones;           // its candidate zones: snapshot groups zone0 .. zone0 + n_zones - 1
    int32_t q_begin, q_end;           // its queue: ZoneFifoIn::queue[q_begin .. q_end)
    int32_t e0, ne, d0, nd;           // az-aware: its undivided orders, entries e0 .. e0+ne-1 / d0 .. d0+nd-1 of the fallback view
};

// ---------------------------------------------------------------------------------------------
// One application, one warp, against an immutable snapshot (GP_MODE_INDEPENDENT; the FIFO modes live in
// gangpack_fifo.cuh).  Returns the driver's node index (>= 0) or -1.
// ALGO: 0 tightly-pack, 1 distribute-evenly.  wcache: this warp's kCapCache x uint16 scratch in shared memory.
// ---------------------------------------------------------------------------------------------
// MUT: the snapshot changes inside the launch (zone-aware FIFO, gangpack_zones.cuh): coherent loads, never with C32 (the
// compact view is not kept current).  grp_override / out_override: pack against another instance group than pa->group and
// write ExecutorNodes (and the candidate list) at another offset than pa->out_off.
// MAP: GroupSlots, or GatherSlots with `view` (tightly-pack over the full-width slots; grp_override and g0 are then unused).
// The gather view takes coherent loads (MUT) inside the FIFO loop and read-only loads in gp_pack_az_fallback, where
// nothing writes the slots.
template <int ALGO, bool FAST, bool NOGPU, bool C32, class OUT, bool MUT = false, class MAP = GroupSlots>
__device__ __forceinline__ int32_t pack_app_impl(const Snapshot& s, const PrepApp* __restrict__ pa,
                                                 OUT* __restrict__ executor_nodes, int2* __restrict__ scratch,
                                                 uint16_t* __restrict__ wcache, WarpStats& st, int lane,
                                                 int snap_flags, const GroupDesc& g0,
                                                 int32_t grp_override = -1, int64_t out_override = -1,
                                                 const MAP* __restrict__ view = nullptr) {
    static_assert(!(MUT && C32), "the compact view is read-only");
    static_assert(!MAP::kGather || (ALGO == 0 && !C32), "the gather scan is tightly-pack over the full-width slots");
    Caps<FAST> a;
    a.init(pa, (pa->flags & kAppUsesGpu) || (snap_flags & kSnapGpuNegative));
    const bool ug = NOGPU ? false : a.use_gpu;      // compile-time false on the hot instantiation
    if (C32) a.init32(s.meta);
    GroupDesc g;
    if constexpr (MAP::kGather) {
        g.sbase = 0; g.ne = view->ne; g.dbase = 0; g.nd = view->nd;   // no group: only the lengths are used
    } else {
        const int32_t grp = grp_override >= 0 ? grp_override : pa->group;
        g = grp == 0 ? g0 : s.groups[grp];                 // group 0's descriptor is kept in registers by the caller
    }
    // slot of executor-order position i
    auto xslot = [&](int32_t i) -> int32_t {
        if constexpr (MAP::kGather) return __ldg(view->exec_slot + i);
        else return g.sbase + i;
    };
    const uint32_t k = a.k;
    const uint32_t lmax = (uint32_t)pa->lmax;
    const int32_t ne = g.ne;
    const int64_t out_off = out_override >= 0 ? out_override : pa->out_off;
    OUT* out = executor_nodes + out_off;
    int2* list = scratch ? scratch + out_off : nullptr;   // distribute-evenly candidate list
    const bool cache_ok = k <= 0xFFFFu;

    // ---- phase 1: how many executors fit, walking the executor priority order --------------------
    // P = sum min(cap(n|0), k) over the scanned prefix; m1 = #nodes with cap >= 1.
    // Early exit is exact: once P >= k + lmax (or m1 >= k+1) every driver candidate that fits
    // leaves >= k executor slots inside the prefix (the driver displaces <= lmax of them, all on one
    // node).  distribute-evenly may only stop on m1 >= k+1 (then one round places everything).
    // Each lane evaluates two nodes per step (64 per warp): two independent 128-bit loads in flight and the
    // vote / reduction / loop control amortised over twice the nodes.
    unsigned long long P = 0;
    uint32_t m1 = 0;
    int32_t pos = 0;
    int32_t first_nz = -1;                    // first step that saw any capacity: emission starts there
    bool early = (k == 0);
    const unsigned long long need = (unsigned long long)k + lmax;
    while (!early && pos < ne) {
        const int32_t i0 = pos + lane, i1 = i0 + kWarp;
        uint32_t c0 = 0u, c1 = 0u;
        if (C32) {                                    // 8-byte records, two shifts + two multiply-highs per node
            if (i0 < ne) c0 = a.cap32(__ldg(s.pair32 + g.sbase + i0));
            if (i1 < ne) c1 = a.cap32(__ldg(s.pair32 + g.sbase + i1));
        } else {
            if (i0 < ne) c0 = a.template cap0<MUT>(s, xslot(i0), ug);
            if (i1 < ne) c1 = a.template cap0<MUT>(s, xslot(i1), ug);
        }
        if (cache_ok && i1 < kCapCache) { wcache[i0] = (uint16_t)c0; wcache[i1] = (uint16_t)c1; }
        const unsigned has0 = __ballot_sync(kFull, c0 != 0), has1 = __ballot_sync(kFull, c1 != 0);
        if (ALGO == 1) {
            // remember the first k nodes that can host at all: (position, cap)
            const unsigned below = (1u << lane) - 1u;
            uint32_t r0 = m1 + __popc(has0 & below);
            uint32_t r1 = m1 + __popc(has0) + __popc(has1 & below);
            if (c0 != 0 && r0 < k) list[r0] = make_int2(i0, (int)c0);
            if (c1 != 0 && r1 < k) list[r1] = make_int2(i1, (int)c1);
        }
        if (first_nz < 0 && (has0 | has1)) first_nz = has0 ? pos : pos + kWarp;
        P += warp_sum(c0 + c1);
        m1 += __popc(has0) + __popc(has1);
        pos += 2 * kWarp;
        if (ALGO == 0) early = (P >= need) || (m1 >= k + 1);
        else early = (m1 >= k + 1);
    }
    st.nodes += (unsigned long long)(pos < ne ? pos : ne);
    const int32_t cached_end = cache_ok ? (pos < kCapCache ? pos : kCapCache) : 0;
    const bool exact_total = !early;          // scanned everything: P == S0
    if (exact_total && P < k) return -1;      // not even without a driver
    if (first_nz < 0) first_nz = 0;

    // ---- phase 2: first feasible driver candidate (binpack.go:67-85) ----------------------------
    // dslot: the driver's executor-order position (>= ne: not an executor candidate); dglob: its slot
    int32_t dslot = -1, dglob = -1;
    for (int32_t j0 = 0; j0 < g.nd && dslot < 0; j0 += kWarp) {
        int32_t j = j0 + lane;
        bool feasible = false;
        int32_t ls = -1, gs = -1;
        if (j < g.nd) {
            if constexpr (MAP::kGather) {
                const int32_t p = __ldg(view->drv_pos + j);
                ls = p < 0 ? ne : p;
                gs = __ldg(view->drv_slot + j);
            } else {
                ls = s.drv_slot[g.dbase + j];
                gs = g.sbase + ls;
            }
            feasible = driver_fits<MUT>(s, gs, a, ug);
            if (feasible && exact_total && ls < ne) {
                // the executor total with the driver on this node must still reach k
                uint32_t c0 = a.template cap0<MUT>(s, gs, ug);
                uint32_t cdl = a.template cap<MUT>(s, gs, a.d_cpu, a.d_mem, a.d_gpu, ug);
                feasible = (P - c0 + cdl >= k);
            }
        }
        unsigned vote = __ballot_sync(kFull, feasible);
        st.drivers += (unsigned long long)((g.nd - j0) < kWarp ? (g.nd - j0) : kWarp);
        if (vote) {
            dslot = __shfl_sync(kFull, ls, __ffs(vote) - 1);
            if constexpr (MAP::kGather) dglob = __shfl_sync(kFull, gs, __ffs(vote) - 1);
        }
    }
    if (dslot < 0) return -1;
    if constexpr (!MAP::kGather) dglob = g.sbase + dslot;
    const int32_t driver_node = s.slot_node[dglob];
    // cap(d | drv): only matters when the driver's node is an executor candidate
    const uint32_t cd = (dslot < ne && k != 0) ? a.template cap<MUT>(s, dglob, a.d_cpu, a.d_mem, a.d_gpu, ug) : 0u;

    // ---- phase 3: emit ExecutorNodes -------------------------------------------------------------
    if (k != 0) {
        if (ALGO == 0) {
            // node-major: node n receives min(cap_d(n), remaining)  (pack_tightly.go:45-61)
            uint32_t placed = 0;
            for (int32_t p0 = first_nz; placed < k && p0 < ne; p0 += kWarp) {   // nodes before first_nz host nothing
                int32_t i = p0 + lane;
                uint32_t c = 0;
                if (i == dslot) c = cd;
                else if (i < cached_end) c = wcache[i];
                else if (i < ne) c = C32 ? a.cap32(__ldg(s.pair32 + g.sbase + i)) : a.template cap0<MUT>(s, xslot(i), ug);
                if (p0 >= cached_end) st.nodes += (unsigned long long)((ne - p0) < kWarp ? (ne - p0) : kWarp);
                uint32_t incl = warp_incl_scan(c, lane);
                uint32_t total = __shfl_sync(kFull, incl, kWarp - 1);
                uint32_t room = k - placed;
                uint32_t T = total < room ? total : room;
                if (T != 0) {
                    uint32_t excl = incl - c;
                    uint32_t take = excl >= T ? 0u : ((c < T - excl) ? c : (T - excl));
                    int32_t node = (take != 0) ? s.slot_node[xslot(i)] : -1;
                    // cooperative expansion: output j belongs to the first lane with incl > j
                    for (uint32_t j = lane; j < ((T + kWarp - 1) & ~(uint32_t)(kWarp - 1)); j += kWarp) {
                        int lo = 0;
#pragma unroll
                        for (int step = 16; step >= 1; step >>= 1) {
                            uint32_t v = __shfl_sync(kFull, incl, lo + step - 1);
                            if (v <= j) lo += step;
                        }
                        int32_t nd = __shfl_sync(kFull, node, lo & 31);
                        if (j < T) out[placed + j] = (OUT)nd;
                    }
                }
                placed += T;
            }
        } else if (early) {
            // one round: the first k nodes with cap_d >= 1, in order  (distribute_evenly.go:49-70)
            uint32_t placed = 0;
            for (int32_t p0 = first_nz; placed < k && p0 < ne; p0 += kWarp) {
                int32_t i = p0 + lane;
                uint32_t c = 0;
                if (i == dslot) c = cd;
                else if (i < cached_end) c = wcache[i];
                else if (i < ne) c = C32 ? a.cap32(__ldg(s.pair32 + g.sbase + i)) : a.template cap0<MUT>(s, g.sbase + i, ug);
                if (p0 >= cached_end) st.nodes += (unsigned long long)((ne - p0) < kWarp ? (ne - p0) : kWarp);
                unsigned has = __ballot_sync(kFull, c != 0);
                uint32_t r = placed + __popc(has & ((1u << lane) - 1u));
                if (c != 0 && r < k) out[r] = (OUT)s.slot_node[g.sbase + i];
                placed += __popc(has);
            }
        } else {
            __syncwarp();
            evenly_rounds<0, OUT>(list, m1, k, dslot, cd, out, s.slot_node + g.sbase, lane, [](int32_t) {});
        }
    }

    return driver_node;
}

// everything that is not (fast class, gpu dimension idle): any int64 request / binding gpu dimension
template <int ALGO, class OUT>
__device__ __noinline__ int32_t pack_app_general(const Snapshot& s, const PrepApp* __restrict__ pa,
                                                 OUT* __restrict__ executor_nodes, int2* __restrict__ scratch,
                                                 uint16_t* __restrict__ wcache, WarpStats& st, int lane, int snap_flags) {
    const GroupDesc g0 = s.groups[0];
    return pack_app_impl<ALGO, false, false, false, OUT>(s, pa, executor_nodes, scratch, wcache, st, lane, snap_flags, g0);
}

// fast class that cannot use the compact view: a cpu or memory request shift 32 or more above the view's shift (a fast
// request never has a shift below it, since max_avail >> sh < 2^32 forces sh >= S).  Such a request exceeds every
// availability of the snapshot, so its capacities here are all 0.
template <int ALGO, class OUT>
__device__ __noinline__ int32_t pack_app_fast64(const Snapshot& s, const PrepApp* __restrict__ pa,
                                                OUT* __restrict__ executor_nodes, int2* __restrict__ scratch,
                                                uint16_t* __restrict__ wcache, WarpStats& st, int lane, int snap_flags) {
    const GroupDesc g0 = s.groups[0];
    return pack_app_impl<ALGO, true, true, false, OUT>(s, pa, executor_nodes, scratch, wcache, st, lane, snap_flags, g0);
}

// class dispatch (warp-uniform): hot path = fast class with the gpu dimension idle
template <int ALGO, class OUT>
__device__ __forceinline__ int32_t pack_app(const Snapshot& s, const PrepApp* __restrict__ pa, OUT* __restrict__ executor_nodes,
                                            int2* __restrict__ scratch, uint16_t* __restrict__ wcache, WarpStats& st, int lane,
                                            int snap_flags, const GroupDesc& g0) {
    const uint32_t fl = pa->flags;
    const bool gpu_idle = !(fl & kAppUsesGpu) && !(snap_flags & kSnapGpuNegative);
    if ((fl & kAppFast32) && gpu_idle)     // hottest path: compact 32-bit snapshot view
        return pack_app_impl<ALGO, true, true, true, OUT>(s, pa, executor_nodes, scratch, wcache, st, lane, snap_flags, g0);
    if ((fl & kAppFast) && gpu_idle)
        return pack_app_fast64<ALGO, OUT>(s, pa, executor_nodes, scratch, wcache, st, lane, snap_flags);
    return pack_app_general<ALGO, OUT>(s, pa, executor_nodes, scratch, wcache, st, lane, snap_flags);
}

// ---------------------------------------------------------------------------------------------
// application preparation (validation bits, division recipes, driver-displacement bound, arithmetic class)
// shared by gp_prep_apps (thread per application) and the fused pack kernels (lanes 0..2 of a warp, one dimension each)
// ---------------------------------------------------------------------------------------------
// One dimension: `bad` gets the validation bits, `l` the bound ceil(d/e) on the executors the driver displaces in this
// dimension, `fast` is cleared when the dimension does not qualify for the 32-bit class.
__device__ __forceinline__ DimDiv prep_dim(int64_t d, int64_t e, int t, long long max_avail, int& bad, uint64_t& l, bool& fast) {
    if (d < 0 || e < 0) bad |= kErrNegativeRequest;
    if (d >= kMaxQuantity || e >= kMaxQuantity) bad |= kErrUnrepresentable;
    DimDiv dv;
    dv.e = e; dv.magic = 0; dv.sh = 0; dv.kind = kDivInf;
    l = 0;
    if (e > 0) {
        const uint32_t sh = (uint32_t)(__ffsll((long long)e) - 1);
        const uint64_t odd = (uint64_t)e >> sh;
        dv.sh = sh;
        if (odd == 1 && sh >= 1) { dv.kind = kDivMagic; dv.magic = 1ull << 63; dv.sh = sh - 1; }   // a / 2^sh = (a >> (sh-1)) / 2
        else if (odd == 1) dv.kind = kDivShift;                                                     // e == 1
        else if ((odd >> 32) == 0) { dv.kind = kDivMagic; dv.magic = 0xFFFFFFFFFFFFFFFFull / odd + 1; }
        else { dv.kind = kDivSlow; dv.sh = 0; }
        if (d > 0) l = ((uint64_t)d + (uint64_t)e - 1) / (uint64_t)e;   // a driver of d displaces at most ceil(d/e) executors here
    }
    // fast class: the shifted numerator of every node fits 32 bits (SnapMeta::max_avail bounds it)
    if (dv.kind == kDivSlow) fast = false;
    else if (t < 2 && dv.kind != kDivMagic) fast = false;       // cpu / mem of the fast class are magic divisions only
    else if (dv.kind != kDivInf) {
        if (max_avail > 0 && (((unsigned long long)max_avail >> dv.sh) >> 32) != 0) fast = false;
    }
    return dv;
}
// compact 32-bit view usable: the request shifts are at least the view's shifts
__device__ __forceinline__ bool prep_fast32(bool fast, const DimDiv& c, const DimDiv& m, const SnapMeta* meta) {
    return fast && c.kind == kDivMagic && m.kind == kDivMagic && (int)c.sh >= meta->shift32[0] && (int)m.sh >= meta->shift32[1] &&
           (int)c.sh - meta->shift32[0] < 32 && (int)m.sh - meta->shift32[1] < 32;   // 32-bit shift amounts
}

}  // namespace gp

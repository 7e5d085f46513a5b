// gangpack_api.cu -- global kernels + the C ABI of include/gangpack.h.
// There is no CPU code path in this library: without a usable CUDA device gp_create fails.
#include "gangpack.h"
#include "gangpack_kernels.cuh"
#include "gangpack_fifo.cuh"
#include "gangpack_minfrag.cuh"
#include "gangpack_tables.cuh"
#include "gangpack_zones.cuh"
#include "gangpack_zonefifo.cuh"
#include "gangpack_resched.cuh"
#include "gangpack_sort.cuh"
#include "gangpack_zonelayout.cuh"
#include "gangpack_reschedprep.cuh"
#include "gangpack_efficiency.cuh"
#include "gangpack_affinity.cuh"
#include "gangpack_capacity.cuh"
#include "gangpack_reconcile.cuh"
#include "gangpack_overhead.cuh"

#include <algorithm>
#include <chrono>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

using namespace gp;

// =============================================================================================
// kernels
// =============================================================================================

constexpr int kPrepThreads = 256;
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

// ---- snapshot construction -------------------------------------------------------------------
__device__ __forceinline__ int32_t find_group(const int32_t* off, int32_t n_groups, int32_t idx) {
    int32_t lo = 0, hi = n_groups - 1;
    while (lo < hi) {
        int32_t mid = (lo + hi + 1) >> 1;
        if (off[mid] <= idx) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// snapshot-wide facts: negative gpu availability, per-dimension maxima (bounds for the fast class).  A CTA of
// gp_build_slots_exec reduces its nodes' values to one SnapPart; every CTA of gp_build_slots_drv folds all parts.
struct SnapPart { long long max_avail[3]; int flags; int pad; };
static_assert(sizeof(SnapPart) == 32, "SnapPart layout");
constexpr int kSnapThreads = 256;       // threads per CTA of both layout kernels
// Block-wide max of (c, m, g) and OR of f, called by every thread of the CTA; the result is valid in thread 0.
__device__ __forceinline__ void block_fold(long long& c, long long& m, long long& g, int& f) {
    __shared__ SnapPart s_part[kSnapThreads / 32];
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        c = max(c, __shfl_xor_sync(kFull, c, d));
        m = max(m, __shfl_xor_sync(kFull, m, d));
        g = max(g, __shfl_xor_sync(kFull, g, d));
        f |= __shfl_xor_sync(kFull, f, d);
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();                    // s_part may still be read by an earlier call
    if (lane == 0) { s_part[w].max_avail[0] = c; s_part[w].max_avail[1] = m; s_part[w].max_avail[2] = g; s_part[w].flags = f; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int t = 1; t < kSnapThreads / 32; ++t) {
            c = max(c, s_part[t].max_avail[0]); m = max(m, s_part[t].max_avail[1]); g = max(g, s_part[t].max_avail[2]);
            f |= s_part[t].flags;
        }
    }
}

// The slot layout is two launches (gp_set_snapshot, gp_set_snapshot_device, gp_prepare_cluster), and no memset: every
// word they leave behind is written by one of them.
// K1 gp_build_slots_exec: thread i writes group descriptor i, lays out executor-order entry i in its slot, scatters
//    drv_pos[node] = i for driver-order entry i, and takes the availability of both entries into its CTA's SnapPart (a
//    node's availability does not depend on its slot); with node_cpu != NULL it also copies node-table entry i into the
//    context's node-table arrays (gp_get_snapshot).  Every CTA writes its part, zeros included, so nothing needs a reset.
// K2 gp_build_slots_drv: every CTA first folds K1's parts (written by the previous launch on the stream: no fence or
//    counter needed) into the maxima its compact views shift by; CTA 0 publishes them in SnapMeta (flags, max_avail,
//    shift32).  Thread s <= n_slots owns slot s.  Executor slots get their compact view; the spare slot of driver-order
//    entry j either receives that node (driver-only) or stays unused (-1: the node has an executor slot in the group);
//    slots past the last group (the orders' lengths may be upper bounds) are -1 as well.  So no slot_node memset is needed.
//    Thread n_slots + 1 + v owns node v: it writes node_slot[v] = -1 when v is in neither order.
// node_slot and drv_pos keep whatever an earlier layout left (garbage after a reallocation), so membership is tested
// against the arrays K1 has just rewritten, with every stale index range-checked before it is followed:
//   v is in the driver order     iff  p = drv_pos[v] lies in [0, drv_off[n_groups]) and drv_order[p] == v;
//   v has executor slot ns       iff  ns = node_slot[v] is an executor slot of its group and slot_node[ns] == v.
// Race freedom of K2: node_slot[v] is written by K1 (executor nodes), by the slot thread of v's driver-order entry
// (driver-only nodes) or by node thread v (nodes in neither order) -- one writer per entry.  The slot thread reads
// node_slot[v] only for its own node, and the node thread only when v is not in the driver order, so neither reads an
// entry another K2 thread writes.  slot_node is read at executor slots only, which K1 wrote and K2 does not touch.
// n_exec / n_drv may be upper bounds of exec_off[n_groups] / drv_off[n_groups] (device-built orders).
__global__ void __launch_bounds__(kSnapThreads) gp_build_slots_exec(int32_t n_exec, int32_t n_drv, int32_t n_groups, int32_t n_nodes,
                                    const int32_t* __restrict__ exec_off, const int32_t* __restrict__ drv_off,
                                    const int32_t* __restrict__ exec_order, const int32_t* __restrict__ drv_order,
                                    const int64_t* __restrict__ cpu, const int64_t* __restrict__ mem, const int64_t* __restrict__ gpu,
                                    GroupDesc* __restrict__ groups, longlong2* __restrict__ pair, int64_t* __restrict__ sgpu,
                                    int32_t* __restrict__ slot_node, int32_t* __restrict__ node_slot, int32_t* __restrict__ drv_pos,
                                    SnapPart* __restrict__ parts,
                                    int64_t* __restrict__ node_cpu, int64_t* __restrict__ node_mem, int64_t* __restrict__ node_gpu) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    long long c = 0, m = 0, gm = 0;      // only positive availabilities raise the maxima
    int neg = 0;
    if (node_cpu && i < n_nodes) {
        node_cpu[i] = cpu[i];
        node_mem[i] = mem[i];
        node_gpu[i] = gpu ? gpu[i] : 0;
    }
    if (i < n_groups) {
        GroupDesc d;
        d.sbase = exec_off[i] + drv_off[i];
        d.ne = exec_off[i + 1] - exec_off[i];
        d.dbase = drv_off[i];
        d.nd = drv_off[i + 1] - drv_off[i];
        groups[i] = d;
    }
    if (i < n_exec && i < exec_off[n_groups]) {
        const int32_t g = find_group(exec_off, n_groups, i);
        const int32_t slot = exec_off[g] + drv_off[g] + (i - exec_off[g]);
        const int32_t node = exec_order[i];
        const int64_t cv = cpu[node], mv = mem[node], gv = gpu ? gpu[node] : 0;
        pair[slot] = make_longlong2(cv, mv);
        sgpu[slot] = gv;
        c = max(c, (long long)cv); m = max(m, (long long)mv); gm = max(gm, (long long)gv); neg |= gv < 0;
        slot_node[slot] = node;
        node_slot[node] = slot;
    }
    if (i < n_drv && i < drv_off[n_groups]) {
        const int32_t node = drv_order[i];
        const long long gv = gpu ? gpu[node] : 0;
        c = max(c, (long long)cpu[node]); m = max(m, (long long)mem[node]); gm = max(gm, gv); neg |= gv < 0;
        drv_pos[node] = i;
    }
    block_fold(c, m, gm, neg);
    if (threadIdx.x == 0) {
        SnapPart p;
        p.max_avail[0] = c; p.max_avail[1] = m; p.max_avail[2] = gm; p.flags = neg ? kSnapGpuNegative : 0; p.pad = 0;
        parts[blockIdx.x] = p;
    }
}

__device__ __forceinline__ int shift_for(long long mx);
__device__ __forceinline__ uint2 compact_pair(longlong2 v, int s0, int s1);

// the group whose slots [exec_off[g] + drv_off[g], exec_off[g+1] + drv_off[g+1]) hold slot s (s below the last group's end)
__device__ __forceinline__ int32_t slot_group(const int32_t* exec_off, const int32_t* drv_off, int32_t n_groups, int32_t s) {
    int32_t lo = 0, hi = n_groups - 1;
    while (lo < hi) {
        const int32_t mid = (lo + hi + 1) >> 1;
        if (exec_off[mid] + drv_off[mid] <= s) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kSnapThreads) gp_build_slots_drv(int32_t n_slots, int32_t n_groups, int32_t n_nodes, int32_t n_drv,
                                   const int32_t* __restrict__ exec_off, const int32_t* __restrict__ drv_off,
                                   const int32_t* __restrict__ drv_order, const int32_t* __restrict__ drv_pos,
                                   const int64_t* __restrict__ cpu, const int64_t* __restrict__ mem, const int64_t* __restrict__ gpu,
                                   longlong2* __restrict__ pair, int64_t* __restrict__ sgpu, int32_t* __restrict__ slot_node,
                                   int32_t* __restrict__ node_slot, int32_t* __restrict__ drv_slot, const SnapPart* __restrict__ parts,
                                   int32_t n_parts, SnapMeta* __restrict__ meta, uint2* __restrict__ pair32) {
    __shared__ long long s_max[2];
    {
        long long c = 0, m = 0, g = 0;
        int f = 0;
        for (int32_t b = threadIdx.x; b < n_parts; b += blockDim.x) {
            const SnapPart p = parts[b];
            c = max(c, p.max_avail[0]); m = max(m, p.max_avail[1]); g = max(g, p.max_avail[2]); f |= p.flags;
        }
        block_fold(c, m, g, f);
        if (threadIdx.x == 0) {
            s_max[0] = c; s_max[1] = m;
            if (blockIdx.x == 0) {
                meta->flags = f; meta->pad = 0;
                meta->max_avail[0] = c; meta->max_avail[1] = m; meta->max_avail[2] = g;
                meta->shift32[0] = shift_for(c); meta->shift32[1] = shift_for(m);
            }
        }
        __syncthreads();
    }
    const int s0 = shift_for(s_max[0]), s1 = shift_for(s_max[1]);
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    const int32_t used = exec_off[n_groups] + drv_off[n_groups];
    if (s > n_slots) {                                       // node v: -1 when it is in neither order
        const int32_t v = s - n_slots - 1;
        if (v > n_nodes) return;
        const int32_t p = drv_pos[v];
        if (p >= 0 && p < drv_off[n_groups] && p < n_drv && drv_order[p] == v) return;
        const int32_t ns = node_slot[v];
        bool exec = false;
        if (ns >= 0 && ns < used) {
            const int32_t g = slot_group(exec_off, drv_off, n_groups, ns);
            exec = ns - (exec_off[g] + drv_off[g]) < exec_off[g + 1] - exec_off[g] && slot_node[ns] == v;
        }
        if (!exec) node_slot[v] = -1;
        return;
    }
    if (s >= used) {                                         // past the last group
        slot_node[s] = -1;
        if (s < n_slots) pair32[s] = make_uint2(0u, 0u);
        return;
    }
    const int32_t g = slot_group(exec_off, drv_off, n_groups, s);
    const int32_t sbase = exec_off[g] + drv_off[g];
    const int32_t ne = exec_off[g + 1] - exec_off[g];
    const int32_t local = s - sbase;
    if (local < ne) {                                        // executor slot, laid out by K1
        pair32[s] = compact_pair(pair[s], s0, s1);
        return;
    }
    const int32_t j = drv_off[g] + (local - ne);
    const int32_t node = drv_order[j];
    const int32_t ns = node_slot[node];
    if (ns >= sbase && ns < sbase + ne && slot_node[ns] == node) {
        drv_slot[j] = ns - sbase;
        slot_node[s] = -1;                                   // unused spare slot
        pair32[s] = make_uint2(0u, 0u);
    } else {
        const longlong2 v = make_longlong2(cpu[node], mem[node]);
        pair[s] = v;
        sgpu[s] = gpu ? gpu[node] : 0;
        pair32[s] = compact_pair(v, s0, s1);
        slot_node[s] = node;
        node_slot[node] = s;             // the node's availability lives in its spare slot (gp_reserve_placements / gp_apply_usage_delta)
        drv_slot[j] = local;
    }
}

// Several small host->device copies in ONE launch: sources are mapped pinned host buffers read
// straight over PCIe (every tiny DMA copy of a chain pays its own fixed latency in stream order).
struct CopyJob { const void* src; void* dst; unsigned long long bytes; };
struct CopyJobs { CopyJob j[8]; int n; };
__global__ void gp_multi_copy(CopyJobs jobs) {
    for (int k = 0; k < jobs.n; ++k) {
        const unsigned long long words = jobs.j[k].bytes >> 2;     // every array here is a multiple of 4 bytes
        const unsigned int* src = static_cast<const unsigned int*>(jobs.j[k].src);
        unsigned int* dst = static_cast<unsigned int*>(jobs.j[k].dst);
        for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < words;
             i += (unsigned long long)gridDim.x * blockDim.x)
            dst[i] = src[i];
    }
}

// After the slots are laid out: the compact view, 8 bytes per slot instead of 16 (negative availability -> 0:
// capacity 0 either way).  Its shifts are the smallest S with max_avail >> S < 2^32; every thread derives them
// from SnapMeta::max_avail, thread 0 publishes them for gp_prep_apps.
__device__ __forceinline__ int shift_for(long long mx) {
    if (mx <= 0) return 0;
    const int bits = 64 - __clzll(mx);
    return bits > 32 ? bits - 32 : 0;
}
__device__ __forceinline__ uint2 compact_pair(longlong2 v, int s0, int s1) {
    uint2 o;
    o.x = v.x < 0 ? 0u : (uint32_t)((unsigned long long)v.x >> s0);
    o.y = v.y < 0 ? 0u : (uint32_t)((unsigned long long)v.y >> s1);
    return o;
}
// the compact view again after a kernel that charged `pair` (FIFO, reservations, usage deltas)
__global__ void gp_fill_pair32(int32_t n_slots, const longlong2* __restrict__ pair, SnapMeta* __restrict__ meta,
                               uint2* __restrict__ pair32) {
    const int s0 = shift_for(meta->max_avail[0]), s1 = shift_for(meta->max_avail[1]);
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) { meta->shift32[0] = s0; meta->shift32[1] = s1; }
    if (i >= n_slots) return;
    pair32[i] = compact_pair(pair[i], s0, s1);
}

// slots -> node-table order (gp_get_snapshot)
__global__ void gp_scatter_slots(int32_t n_slots, const longlong2* __restrict__ pair, const int64_t* __restrict__ sgpu,
                                 const int32_t* __restrict__ slot_node,
                                 int64_t* __restrict__ cpu, int64_t* __restrict__ mem, int64_t* __restrict__ gpu) {
    int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    int32_t node = slot_node[s];
    if (node < 0) return;
    longlong2 v = pair[s];
    cpu[node] = v.x; mem[node] = v.y; gpu[node] = sgpu[s];
}

// =============================================================================================
// host side
// =============================================================================================

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

// One staging layout in one DevBuf: take() every piece (256-byte-aligned offsets), then reserve() once.
struct Arena {
    DevBuf& buf;
    size_t size = 0;
    size_t take(size_t bytes) { const size_t o = size; size += (bytes + 255) & ~(size_t)255; return o; }
    cudaError_t reserve() { return buf.reserve(size); }
    char* base() const { return buf.as<char>(); }
    cudaError_t upload(size_t off, const void* src, size_t bytes, cudaStream_t st) const {
        return cudaMemcpyAsync(base() + off, src, bytes, cudaMemcpyHostToDevice, st);
    }
};

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
    bool have_snapshot = false;
    int32_t n_nodes = 0, n_groups = 0, n_exec = 0, n_drv = 0, n_slots = 0;
    DevBuf node_cpu, node_mem, node_gpu;        // node-table order (as given)
    DevBuf exec_off, drv_off, exec_order, drv_order;
    DevBuf pair, pair32, sgpu, slot_node, node_slot, drv_slot, groups, snap_flags;
    DevBuf drv_pos;                             // node -> driver-order position, scattered by the layout (gp_build_slots_exec)
    DevBuf snap_part;                           // SnapPart per CTA of gp_build_slots_exec

    // batch staging; a_rows: the six quantity rows in one pitched block (pack_batch_impl)
    DevBuf a_rows, a_count, a_group, a_skip, a_off;
    DevBuf prep, r_driver, r_exec, scratch, dev_misc, gmin, sortbuf, usagebuf, reschedbuf;
    void* pinned_misc = nullptr;                  // PinnedStatus
    DevStatus* status() const { return dev_misc.as<DevStatus>(); }
    PinnedStatus* host_status() const { return static_cast<PinnedStatus*>(pinned_misc); }
    std::vector<int64_t> host_off;
    std::vector<int32_t> v_owner;                 // gp_set_snapshot validation scratch (no per-call allocation)
    // gp_set_snapshot's host copy of the layout, kept for gp_pack_fifo_az_aware's order checks: v_owner[v] (group, roles)
    // and v_pos[v] / v_pos[n_nodes + v] (position of v in its group's executor / driver order).  host_layout: they
    // describe the current snapshot (false after gp_set_snapshot_device / gp_prepare_cluster or a refused gp_set_snapshot)
    std::vector<int32_t> v_pos;
    bool host_layout = false;
    std::vector<uint8_t> v_seen_e, v_seen_d;
    std::vector<int32_t> v_zone_next;             // az-aware order check: next position per zone group
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
    bool have_sched = false;
    // SchedulableResources for gp_packing_efficiency alone: also set by gp_prepare_cluster, whose one-group snapshot the zone
    // entry points keep refusing (have_sched stays false there)
    bool have_eff_sched = false;
    // gp_prepare_cluster_zones: the undivided orders it sorted (in zoneprep, which also holds that call's scratch), their
    // lengths and n_zones as DEVICE pointers for gp_pack_*_az_aware(orders == NULL); zone_kind = the gp_zone_layout_kind of the
    // current snapshot, -1 when another entry laid it out
    DevBuf zoneprep;
    DevBuf reschedprep;                           // gp_reschedule_from_reservations' own scratch (no state points into it)
    DevBuf capprep;                               // gp_exceeds_cluster_capacity's own scratch (no state points into it)
    DevBuf reconbuf;                              // gp_reconcile_find_nodes' own scratch (no state points into it)
    DevBuf overbuf;                               // gp_node_overhead's own scratch (no state points into it)
    int zone_kind = -1;
    gp_az_orders zone_orders{};
    bool sort_attr_set = false;
    bool recon_attr_set = false;                  // dynamic shared-memory opt-in of gp_sort_tiles<ReconKey> done on this device
    bool fifo_attr_set[2] = {false, false};       // dynamic shared-memory opt-in of gp_pack_fifo_cta<ALGO,*> done on this device

    gp_stats last{};
};

static thread_local std::string g_create_error;

static cudaError_t create_aux(gp_ctx* c) {
    cudaError_t e;
    for (auto& l : c->lane) if ((e = cudaStreamCreateWithFlags(&l, cudaStreamNonBlocking)) != cudaSuccess) return e;
    for (auto& row : c->ev) for (auto& ev : row) if ((e = cudaEventCreate(&ev)) != cudaSuccess) return e;
    if ((e = cudaEventCreateWithFlags(&c->ev_ready, cudaEventDisableTiming)) != cudaSuccess) return e;
    if ((e = cudaEventCreate(&c->ev_t0)) != cudaSuccess) return e;
    for (auto& ev : c->ev_done) if ((e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return e;
    return cudaSuccess;
}

#define GP_CUDA(ctx, expr)                                                                     \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            (ctx)->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                   \
            return GP_ERR_CUDA;                                                                \
        }                                                                                      \
    } while (0)

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

// Device-visible alias of a host buffer, or nullptr.  Buffers from gp_alloc_pinned are known; anything
// else is asked of the driver (cudaHostRegister / cudaHostAlloc memory of the caller qualifies).
static const void* mapped_ptr(gp_ctx* c, const void* p, size_t bytes) {
    if (!p || !c->zero_copy) return nullptr;
    const char* q = static_cast<const char*>(p);
    for (const auto& b : c->pinned_blocks)
        if (q >= b.first && q + bytes <= b.first + b.second) return p;     // UVA: same address on the device
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (a.type == cudaMemoryTypeHost && a.devicePointer) return a.devicePointer;
    return nullptr;
}

static gp_status fail(gp_ctx* ctx, gp_status st, const std::string& msg) {
    ctx->err = msg;
    return st;
}

static Snapshot make_snapshot(const gp_ctx* c) {
    Snapshot s;
    s.pair = c->pair.as<longlong2>();
    s.pair32 = c->pair32.as<uint2>();
    s.gpu = c->sgpu.as<int64_t>();
    s.slot_node = c->slot_node.as<int32_t>();
    s.drv_slot = c->drv_slot.as<int32_t>();
    s.groups = c->groups.as<GroupDesc>();
    s.meta = c->snap_flags.as<SnapMeta>();
    s.gmins = nullptr;
    s.n_groups = c->n_groups;
    s.n_slots = c->n_slots;
    return s;
}

extern "C" {

int gp_abi_version(void) { return GP_ABI_VERSION; }

const char* gp_last_error(const gp_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int gp_backend(const gp_ctx* ctx) { return ctx ? 1 : 0; }

gp_status gp_create(gp_ctx** out, const gp_config* cfg) {
    if (!out) { g_create_error = "gp_create: out is NULL"; return GP_ERR_INVALID; }
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        g_create_error = std::string("gp_create: no CUDA device (") + cudaGetErrorString(e) +
                         "); libgangpack has no CPU path";
        return GP_ERR_NO_DEVICE;
    }
    int dev = (cfg && cfg->device >= 0) ? cfg->device : -1;
    if (dev < 0) { if (cudaGetDevice(&dev) != cudaSuccess) dev = 0; }
    if (dev >= n) { g_create_error = "gp_create: device ordinal out of range"; return GP_ERR_INVALID; }
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, dev)) != cudaSuccess) {
        g_create_error = std::string("gp_create: cudaGetDeviceProperties: ") + cudaGetErrorString(e);
        return GP_ERR_CUDA;
    }
    if (prop.major != 9 || prop.minor != 0) {
        g_create_error = "gp_create: device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor) +
                         "; this library ships sm_90a code only";
        return GP_ERR_NO_DEVICE;
    }
    gp_ctx* c = new (std::nothrow) gp_ctx();
    if (!c) { g_create_error = "gp_create: out of memory"; return GP_ERR_INVALID; }
    c->device = dev;
    c->sm_count = prop.multiProcessorCount;
    c->async_snapshot = cfg && (cfg->flags & GP_CFG_ASYNC_SNAPSHOT);
    if (const char* z = std::getenv("GANGPACK_ZERO_COPY")) c->zero_copy = std::atoi(z);
    if (const char* z = std::getenv("GANGPACK_TABLES")) c->use_tables = std::atoi(z);
    if (const char* z = std::getenv("GANGPACK_FIFO_WARP")) c->fifo_warp = std::atoi(z);
    if (const char* z = std::getenv("GANGPACK_GRAPHS")) c->use_graphs = std::atoi(z);
    if (const char* z = std::getenv("GANGPACK_CHUNK_APPS")) c->chunk_apps = std::max(1024, std::atoi(z));
    if (const char* z = std::getenv("GANGPACK_TRACE")) c->trace = std::atoi(z);
    if ((e = cudaSetDevice(dev)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = create_aux(c)) != cudaSuccess ||
        (e = cudaHostAlloc(&c->pinned_misc, sizeof(PinnedStatus), cudaHostAllocDefault)) != cudaSuccess ||
        (e = c->dev_misc.reserve(sizeof(DevStatus))) != cudaSuccess || (e = c->snap_flags.reserve(sizeof(SnapMeta))) != cudaSuccess ||
        // the layout writes every SnapMeta word but the padding
        (e = cudaMemsetAsync(c->snap_flags.p, 0, sizeof(SnapMeta), c->stream)) != cudaSuccess ||
        (e = cudaStreamSynchronize(c->stream)) != cudaSuccess) {
        g_create_error = std::string("gp_create: ") + cudaGetErrorString(e);
        delete c;
        return GP_ERR_CUDA;
    }
    *out = c;
    return GP_OK;
}

void gp_destroy(gp_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->pinned_misc) cudaFreeHost(c->pinned_misc);
    if (c->one_block) cudaFreeHost(c->one_block);
    for (auto& row : c->ev) for (cudaEvent_t e : row) if (e) cudaEventDestroy(e);
    if (c->ev_ready) cudaEventDestroy(c->ev_ready);
    if (c->ev_t0) cudaEventDestroy(c->ev_t0);
    for (cudaEvent_t e : c->ev_done) if (e) cudaEventDestroy(e);
    for (cudaStream_t l : c->lane) if (l) cudaStreamDestroy(l);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;                            // device buffers and graphs free themselves
}

gp_status gp_alloc_pinned(gp_ctx* ctx, size_t bytes, void** out) {
    if (!ctx || !out) return GP_ERR_INVALID;
    GP_CUDA(ctx, cudaSetDevice(ctx->device));
    GP_CUDA(ctx, cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocPortable | cudaHostAllocMapped));   // pinned for every device of the process (gp_multi)
    ctx->pinned_blocks.emplace_back(static_cast<const char*>(*out), bytes ? bytes : 1);
    return GP_OK;
}

gp_status gp_free_pinned(gp_ctx* ctx, void* p) {
    if (!ctx) return GP_ERR_INVALID;
    if (p) {
        for (size_t i = 0; i < ctx->pinned_blocks.size(); ++i)
            if (ctx->pinned_blocks[i].first == static_cast<const char*>(p)) { ctx->pinned_blocks.erase(ctx->pinned_blocks.begin() + (long)i); break; }
        GP_CUDA(ctx, cudaFreeHost(p));
    }
    return GP_OK;
}

gp_status gp_register_host(gp_ctx* ctx, void* p, size_t bytes) {
    if (!ctx || !p || !bytes) return GP_ERR_INVALID;
    GP_CUDA(ctx, cudaSetDevice(ctx->device));
    GP_CUDA(ctx, cudaHostRegister(p, bytes, cudaHostRegisterPortable | cudaHostRegisterMapped));
    return GP_OK;
}

gp_status gp_unregister_host(gp_ctx* ctx, void* p) {
    if (!ctx || !p) return GP_ERR_INVALID;
    GP_CUDA(ctx, cudaSetDevice(ctx->device));
    GP_CUDA(ctx, cudaHostUnregister(p));
    return GP_OK;
}

void* gp_stream(gp_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

gp_status gp_synchronize(gp_ctx* ctx) {
    if (!ctx) return GP_ERR_INVALID;
    GP_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GP_OK;
}

}  // extern "C"

// ---- snapshot ---------------------------------------------------------------------------------

// Build the slot layout from DEVICE-resident gp_nodes arrays on `st`.  copy_nodes: the layout kernel also copies the node
// table into node_cpu / node_mem / node_gpu (reserved by the caller; false when dn already points at them).
static gp_status build_snapshot_device(gp_ctx* c, const gp_nodes* dn, int32_t n_exec, int32_t n_drv, cudaStream_t st,
                                       bool copy_nodes = false) {
    const int32_t n_slots = n_exec + n_drv;
    c->host_layout = false;              // gp_set_snapshot sets it again once the layout it validated is in place
    c->zone_kind = -1;                   // gp_prepare_cluster_zones sets it again once its layout is in place
    GP_CUDA(c, c->pair.reserve(sizeof(longlong2) * (size_t)(n_slots + 1)));
    GP_CUDA(c, c->pair32.reserve(sizeof(uint2) * (size_t)(n_slots + 1)));
    GP_CUDA(c, c->sgpu.reserve(sizeof(int64_t) * (size_t)(n_slots + 1)));
    GP_CUDA(c, c->slot_node.reserve(sizeof(int32_t) * (size_t)(n_slots + 1)));
    GP_CUDA(c, c->node_slot.reserve(sizeof(int32_t) * (size_t)(dn->n_nodes + 1)));
    GP_CUDA(c, c->drv_slot.reserve(sizeof(int32_t) * (size_t)(n_drv + 1)));
    GP_CUDA(c, c->groups.reserve(sizeof(GroupDesc) * (size_t)dn->n_groups));
    GP_CUDA(c, c->drv_pos.reserve(sizeof(int32_t) * (size_t)(dn->n_nodes + 1)));
    int64_t* node_cpu = copy_nodes ? c->node_cpu.as<int64_t>() : nullptr;
    const int T = kSnapThreads;
    const int32_t n1 = std::max(std::max(std::max(n_exec, n_drv), dn->n_groups), node_cpu ? dn->n_nodes : 0);
    const int32_t blocks1 = (n1 + T - 1) / T;
    GP_CUDA(c, c->snap_part.reserve(sizeof(SnapPart) * (size_t)blocks1));
    SnapPart* parts = c->snap_part.as<SnapPart>();
    struct { gp_nodes dn; int32_t n_exec, n_drv; void* buf[13]; } key{};
    key.dn = *dn; key.n_exec = n_exec; key.n_drv = n_drv;
    void* bufs[13] = {c->pair.p, c->pair32.p, c->sgpu.p, c->slot_node.p, c->node_slot.p, c->drv_slot.p, c->groups.p, c->snap_flags.p,
                      node_cpu, c->node_mem.p, c->node_gpu.p, c->drv_pos.p, c->snap_part.p};
    std::memcpy(key.buf, bufs, sizeof(bufs));
    gp_status rs = run_cached(c, c->g_snapshot, &key, sizeof(key), st, [&](int& launches) -> gp_status {
        gp_build_slots_exec<<<blocks1, T, 0, st>>>(
            n_exec, n_drv, dn->n_groups, dn->n_nodes, dn->exec_off, dn->drv_off, dn->exec_order, dn->drv_order, dn->avail_cpu_milli,
            dn->avail_mem_bytes, dn->avail_gpu, c->groups.as<GroupDesc>(), c->pair.as<longlong2>(), c->sgpu.as<int64_t>(),
            c->slot_node.as<int32_t>(), c->node_slot.as<int32_t>(), c->drv_pos.as<int32_t>(), parts, node_cpu,
            c->node_mem.as<int64_t>(), c->node_gpu.as<int64_t>());
        // threads [0, n_slots]: slots; [n_slots + 1, n_slots + 1 + n_nodes]: nodes
        gp_build_slots_drv<<<(n_slots + dn->n_nodes + 1 + T) / T, T, 0, st>>>(
            n_slots, dn->n_groups, dn->n_nodes, n_drv, dn->exec_off, dn->drv_off, dn->drv_order, c->drv_pos.as<int32_t>(),
            dn->avail_cpu_milli, dn->avail_mem_bytes, dn->avail_gpu, c->pair.as<longlong2>(), c->sgpu.as<int64_t>(),
            c->slot_node.as<int32_t>(), c->node_slot.as<int32_t>(), c->drv_slot.as<int32_t>(), parts, blocks1,
            c->snap_flags.as<SnapMeta>(), c->pair32.as<uint2>());
        GP_CUDA(c, cudaGetLastError());
        launches = 0;       // (the snapshot layout is not part of a pack call's launch count)
        return GP_OK;
    });
    if (rs != GP_OK) return rs;
    c->n_nodes = dn->n_nodes; c->n_groups = dn->n_groups; c->n_exec = n_exec; c->n_drv = n_drv; c->n_slots = n_slots;
    c->have_snapshot = true;
    c->have_sched = false;               // SchedulableResources belong to a node table
    c->have_eff_sched = false;
    return GP_OK;
}

extern "C" {

gp_status gp_set_snapshot(gp_ctx* c, const gp_nodes* n) {
    if (!c) return GP_ERR_INVALID;
    if (!n || n->n_nodes < 0 || n->n_groups < 1 || !n->exec_off || !n->drv_off ||
        (n->n_nodes > 0 && (!n->avail_cpu_milli || !n->avail_mem_bytes)))
        return fail(c, GP_ERR_INVALID, "gp_set_snapshot: missing arrays or bad sizes");
    // ---- host validation (O(N)): offsets monotone, indices in range, one group per node, domain
    const int32_t G = n->n_groups;
    if (n->exec_off[0] != 0 || n->drv_off[0] != 0) return fail(c, GP_ERR_INVALID, "gp_set_snapshot: offsets must start at 0");
    for (int32_t g = 0; g < G; ++g)
        if (n->exec_off[g + 1] < n->exec_off[g] || n->drv_off[g + 1] < n->drv_off[g])
            return fail(c, GP_ERR_INVALID, "gp_set_snapshot: offsets not monotone");
    const int32_t n_exec = n->exec_off[G], n_drv = n->drv_off[G];
    if ((n_exec > 0 && !n->exec_order) || (n_drv > 0 && !n->drv_order))
        return fail(c, GP_ERR_INVALID, "gp_set_snapshot: order arrays missing");
    {
        // owner[v] = 4 * group + (bit0: listed as executor candidate, bit1: listed as driver candidate); -1 = unseen
        c->host_layout = false;
        std::vector<int32_t>& owner = c->v_owner;
        owner.assign((size_t)n->n_nodes, -1);
        const uint32_t N = (uint32_t)n->n_nodes;
        c->v_pos.resize(2 * (size_t)N);
        int32_t* pos = c->v_pos.data();
        for (int32_t g = 0; g < G; ++g) {
            for (int32_t e = n->exec_off[g]; e < n->exec_off[g + 1]; ++e) {
                const uint32_t v = (uint32_t)n->exec_order[e];
                if (v >= N) return fail(c, GP_ERR_INVALID, "gp_set_snapshot: exec_order index out of range");
                if (owner[v] >= 0) return fail(c, GP_ERR_INVALID, "gp_set_snapshot: node listed twice in executor orders");
                owner[v] = 4 * g + 1;
                pos[v] = e - n->exec_off[g];
            }
        }
        for (int32_t g = 0; g < G; ++g) {
            for (int32_t d = n->drv_off[g]; d < n->drv_off[g + 1]; ++d) {
                const uint32_t v = (uint32_t)n->drv_order[d];
                if (v >= N) return fail(c, GP_ERR_INVALID, "gp_set_snapshot: drv_order index out of range");
                const int32_t o = owner[v];
                if (o >= 0 && (o & 2)) return fail(c, GP_ERR_INVALID, "gp_set_snapshot: node listed twice in driver orders");
                if (o >= 0 && (o >> 2) != g) return fail(c, GP_ERR_INVALID, "gp_set_snapshot: node belongs to two instance groups");
                owner[v] = 4 * g + (o >= 0 ? (o & 3) : 0) + 2;
                pos[N + v] = d - n->drv_off[g];
            }
        }
        // exact-int64 domain: branch-free so that the loop vectorises
        const int64_t* cols[3] = {n->avail_cpu_milli, n->avail_mem_bytes, n->avail_gpu};
        uint64_t out_of_domain = 0;
        for (int k = 0; k < 3; ++k) {
            const int64_t* p = cols[k];
            if (!p) continue;
            for (uint32_t i = 0; i < N; ++i) out_of_domain |= (uint64_t)(p[i] >= kMaxQuantity) | (uint64_t)(p[i] <= -kMaxQuantity);
        }
        if (out_of_domain) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_set_snapshot: |quantity| >= 2^61");
    }
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t nb = sizeof(int64_t) * (size_t)(n->n_nodes + 1);
    GP_CUDA(c, c->node_cpu.reserve(nb)); GP_CUDA(c, c->node_mem.reserve(nb)); GP_CUDA(c, c->node_gpu.reserve(nb));
    GP_CUDA(c, c->exec_off.reserve(sizeof(int32_t) * (size_t)(G + 1)));
    GP_CUDA(c, c->drv_off.reserve(sizeof(int32_t) * (size_t)(G + 1)));
    GP_CUDA(c, c->exec_order.reserve(sizeof(int32_t) * (size_t)(n_exec + 1)));
    GP_CUDA(c, c->drv_order.reserve(sizeof(int32_t) * (size_t)(n_drv + 1)));
    const size_t vb = sizeof(int64_t) * (size_t)n->n_nodes;
    const size_t ob = sizeof(int32_t) * (size_t)(G + 1);
    // mapped pinned inputs: one gather-copy kernel reads them over PCIe instead of 7 chained DMA copies
    const void* m_cpu = mapped_ptr(c, n->avail_cpu_milli, vb);
    const void* m_mem = mapped_ptr(c, n->avail_mem_bytes, vb);
    const void* m_gpu = n->avail_gpu ? mapped_ptr(c, n->avail_gpu, vb) : nullptr;
    const void* m_eoff = mapped_ptr(c, n->exec_off, ob);
    const void* m_doff = mapped_ptr(c, n->drv_off, ob);
    const void* m_eord = n_exec ? mapped_ptr(c, n->exec_order, sizeof(int32_t) * (size_t)n_exec) : n->exec_order;
    const void* m_dord = n_drv ? mapped_ptr(c, n->drv_order, sizeof(int32_t) * (size_t)n_drv) : n->drv_order;
    const bool all_mapped = vb && m_cpu && m_mem && (!n->avail_gpu || m_gpu) && m_eoff && m_doff && (!n_exec || m_eord) && (!n_drv || m_dord);
    if (all_mapped) {
        CopyJobs jobs{};
        auto add = [&](const void* src, void* dst, size_t bytes) { if (bytes) jobs.j[jobs.n++] = CopyJob{src, dst, bytes}; };
        add(m_cpu, c->node_cpu.p, vb); add(m_mem, c->node_mem.p, vb);
        if (n->avail_gpu) add(m_gpu, c->node_gpu.p, vb);
        add(m_eoff, c->exec_off.p, ob); add(m_doff, c->drv_off.p, ob);
        add(m_eord, c->exec_order.p, sizeof(int32_t) * (size_t)n_exec);
        add(m_dord, c->drv_order.p, sizeof(int32_t) * (size_t)n_drv);
        if (!n->avail_gpu) GP_CUDA(c, cudaMemsetAsync(c->node_gpu.p, 0, vb, st));
        gp_multi_copy<<<c->sm_count, 512, 0, st>>>(jobs);
        GP_CUDA(c, cudaGetLastError());
    } else {
        if (vb) {
            GP_CUDA(c, cudaMemcpyAsync(c->node_cpu.p, n->avail_cpu_milli, vb, cudaMemcpyHostToDevice, st));
            GP_CUDA(c, cudaMemcpyAsync(c->node_mem.p, n->avail_mem_bytes, vb, cudaMemcpyHostToDevice, st));
            if (n->avail_gpu) GP_CUDA(c, cudaMemcpyAsync(c->node_gpu.p, n->avail_gpu, vb, cudaMemcpyHostToDevice, st));
            else GP_CUDA(c, cudaMemsetAsync(c->node_gpu.p, 0, vb, st));
        }
        GP_CUDA(c, cudaMemcpyAsync(c->exec_off.p, n->exec_off, ob, cudaMemcpyHostToDevice, st));
        GP_CUDA(c, cudaMemcpyAsync(c->drv_off.p, n->drv_off, ob, cudaMemcpyHostToDevice, st));
        if (n_exec) GP_CUDA(c, cudaMemcpyAsync(c->exec_order.p, n->exec_order, sizeof(int32_t) * (size_t)n_exec, cudaMemcpyHostToDevice, st));
        if (n_drv) GP_CUDA(c, cudaMemcpyAsync(c->drv_order.p, n->drv_order, sizeof(int32_t) * (size_t)n_drv, cudaMemcpyHostToDevice, st));
    }
    gp_nodes dn = *n;
    dn.avail_cpu_milli = c->node_cpu.as<int64_t>(); dn.avail_mem_bytes = c->node_mem.as<int64_t>();
    dn.avail_gpu = c->node_gpu.as<int64_t>();
    dn.exec_off = c->exec_off.as<int32_t>(); dn.drv_off = c->drv_off.as<int32_t>();
    dn.exec_order = c->exec_order.as<int32_t>(); dn.drv_order = c->drv_order.as<int32_t>();
    gp_status s = build_snapshot_device(c, &dn, n_exec, n_drv, st);
    if (s != GP_OK) return s;
    c->host_layout = true;
    // GP_CFG_ASYNC_SNAPSHOT with page-locked inputs: return while the device is still reading them -- the upload and the
    // slot layout then overlap the H2D copies of the gp_pack_* call that follows
    if (!(c->async_snapshot && all_mapped)) GP_CUDA(c, cudaStreamSynchronize(st));   // the caller may reuse its host buffers
    return GP_OK;
}

gp_status gp_set_snapshot_device(gp_ctx* c, const gp_nodes* dn, int32_t n_exec, int32_t n_drv, void* stream) {
    if (!c) return GP_ERR_INVALID;
    if (!dn || dn->n_nodes < 0 || dn->n_groups < 1 || !dn->exec_off || !dn->drv_off || n_exec < 0 || n_drv < 0 ||
        (n_exec > 0 && !dn->exec_order) || (n_drv > 0 && !dn->drv_order))
        return fail(c, GP_ERR_INVALID, "gp_set_snapshot_device: missing arrays or bad sizes");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream;
    // keep a node-table copy so gp_get_snapshot can answer for nodes outside every group: the layout kernel makes it
    const size_t nb = sizeof(int64_t) * (size_t)(dn->n_nodes + 1);
    GP_CUDA(c, c->node_cpu.reserve(nb)); GP_CUDA(c, c->node_mem.reserve(nb)); GP_CUDA(c, c->node_gpu.reserve(nb));
    return build_snapshot_device(c, dn, n_exec, n_drv, st, dn->n_nodes > 0);
}

gp_status gp_get_snapshot(gp_ctx* c, int64_t* cpu, int64_t* mem, int64_t* gpu) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_get_snapshot: no snapshot");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const int T = 256;
    if (c->n_slots > 0)
        gp_scatter_slots<<<(c->n_slots + T - 1) / T, T, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), c->sgpu.as<int64_t>(),
                                                                c->slot_node.as<int32_t>(), c->node_cpu.as<int64_t>(),
                                                                c->node_mem.as<int64_t>(), c->node_gpu.as<int64_t>());
    GP_CUDA(c, cudaGetLastError());
    const size_t vb = sizeof(int64_t) * (size_t)c->n_nodes;
    if (vb) {
        if (cpu) GP_CUDA(c, cudaMemcpyAsync(cpu, c->node_cpu.p, vb, cudaMemcpyDeviceToHost, st));
        if (mem) GP_CUDA(c, cudaMemcpyAsync(mem, c->node_mem.p, vb, cudaMemcpyDeviceToHost, st));
        if (gpu) GP_CUDA(c, cudaMemcpyAsync(gpu, c->node_gpu.p, vb, cudaMemcpyDeviceToHost, st));
    }
    GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

}  // extern "C"

// ---- packing ------------------------------------------------------------------------------------

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
                               volatile int* err_host, bool use_tables, int64_t seg_bound, unsigned int* status_zero, cudaStream_t st) {
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
    gp_decide_tables<ALGO, OUT><<<(int)blocks, kTabThreads, 0, st>>>(s, cols, tabs, off_base, off_out, app_slot, q, dr.cap, dr.driver + lo,
                                                                    static_cast<OUT*>(dr.exec), prep, listed, stats, d_err, err_host,
                                                                    use_tables ? 0 : 1, status_zero);
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
    // it also zeroes the classify tiles' and the table segments' look-back words (see there)
    gp_pack_listed<ALGO, OUT><<<(int)blocks, kPackTabThreads, 0, st>>>(s, tabs, (int32_t)tiles, use_tables ? kMaxShapes * (int32_t)seg_bound : 0,
                                                                      prep, listed, dr.driver + lo, static_cast<OUT*>(dr.exec), scratch,
                                                                      stats, next_app);
    c->last.kernel_launches += 2;
    return GP_OK;
}

// Device-resident apps [lo, hi): enqueue the kernels on `st`; chunk index selects the timing events and the table lane.
// off_base: ExecutorNodes offset of application `lo` (only used when the offsets are derived on the device).
// status_in_kernel: pack_begin left the status block to this range's decide kernel (kernel_zeroes_status(), one range only).
static gp_status pack_device_range(gp_ctx* c, const DevApps& da, int32_t lo, int32_t hi, int64_t off_base, gp_algo algo, gp_mode mode,
                                   const DevResults& dr, int2* scratch, cudaStream_t st, int chunk, bool status_in_kernel = false) {
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
        GP_CUDA(c, T.hdr.reserve_zeroed(hdr_bytes, st));
        // [executor slot | driver slot | listed]
        GP_CUDA(c, T.app_slot.reserve(sizeof(int32_t) * (3 * (size_t)q + 1)));
        if (use_tables) {
            GP_CUDA(c, T.table.reserve(sizeof(uint32_t) * (size_t)kMaxShapes * (size_t)((c->n_slots + 4) & ~3)));
            // total | firstfit | first_host | segments before each group
            GP_CUDA(c, T.total.reserve(sizeof(uint32_t) * (3 * (size_t)kMaxShapes * (size_t)c->n_groups + (size_t)c->n_groups + 1)));
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
        tabs.seg_pre = tabs.first_host + (size_t)kMaxShapes * (size_t)c->n_groups;
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
                                       d_err, err_host, use_tables, seg_bound, status_zero, st);
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
        struct { int32_t algo, o16, use_tables, q, lo, chunk; int64_t off_base; AppColumns cols; ShapeTables tabs; Snapshot snap;
                 const void* p[11]; int64_t cap; } key{};
        key.algo = (int32_t)algo; key.o16 = o16; key.use_tables = use_tables; key.q = q; key.lo = lo; key.chunk = chunk; key.off_base = off_base;
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
static gp_status pack_begin(gp_ctx* c, int32_t q, gp_algo algo, gp_mode mode, int64_t exec_cap, bool derive_off, int2** scratch, cudaStream_t st,
                            bool status_in_kernel = false) {
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
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, std::string(who) + ": gp_set_snapshot first");
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
static gp_status host_error(gp_ctx* c) { return decode_device_error(c, c->host_status()->err_word); }

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
    if (!c) return GP_ERR_INVALID;
    if (!da || !dout) return fail(c, GP_ERR_INVALID, "gp_pack_batch_device: NULL apps/results");
    const gp_apps_wire w = widen(da);
    gp_results_wire ow{dout->driver_node, dout->executor_nodes, dout->executor_nodes_cap, 32, 0};
    gp_status s = check_args(c, &w, algo, mode, &ow, "gp_pack_batch_device");
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream;
    int2* scratch = nullptr;
    const bool zero_in_kernel = kernel_zeroes_status(w.n_apps, algo, mode);
    s = pack_begin(c, w.n_apps, algo, mode, ow.executor_nodes_cap, !w.exec_out_off, &scratch, st, zero_in_kernel);
    if (s != GP_OK || w.n_apps == 0) return s;
    DevApps dv{};
    dv.cols.q[0] = w.drv_cpu; dv.cols.q[1] = w.drv_mem; dv.cols.q[2] = w.drv_gpu;
    dv.cols.q[3] = w.exe_cpu; dv.cols.q[4] = w.exe_mem; dv.cols.q[5] = w.exe_gpu;
    dv.cols.count = w.exe_count; dv.cols.group = w.group; dv.cols.off = w.exec_out_off; dv.cols.bits = 64; dv.cols.mem_shift = 0;
    dv.skip = w.skip_if_no_fit; dv.n = w.n_apps;
    DevResults dr{ow.driver_node, ow.executor_nodes, ow.executor_nodes_cap, 32};
    s = pack_device_range(c, dv, 0, w.n_apps, 0, algo, mode, dr, scratch, st, 0, zero_in_kernel);
    if (s == GP_OK) c->ev_chunks = 1;
    return s;
}

gp_status gp_last_stats(gp_ctx* c, gp_stats* out) {
    if (!c || !out) return GP_ERR_INVALID;
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
    if (!c) return GP_ERR_INVALID;
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
    if (!c) return GP_ERR_INVALID;
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

// ---- single-AZ packers: pack every zone, choose by packing efficiency on the device (gangpack_zones.cuh) ----------
gp_status gp_set_schedulable(gp_ctx* c, const int64_t* cpu, const int64_t* mem, const int64_t* gpu) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_set_schedulable: gp_set_snapshot first");
    if (c->n_nodes > 0 && (!cpu || !mem)) return fail(c, GP_ERR_INVALID, "gp_set_schedulable: missing arrays");
    GP_CUDA(c, cudaSetDevice(c->device));
    const size_t N = (size_t)c->n_nodes;
    for (size_t i = 0; i < N; ++i) {
        const int64_t v[3] = {cpu[i], mem[i], gpu ? gpu[i] : 0};
        for (int64_t x : v) if (x >= kMaxQuantity || x <= -kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_set_schedulable: |quantity| >= 2^61");
    }
    GP_CUDA(c, c->sched.reserve(24 * (N + 1)));
    char* b = c->sched.as<char>();
    if (N) {
        GP_CUDA(c, cudaMemcpyAsync(b, cpu, 8 * N, cudaMemcpyHostToDevice, c->stream));
        GP_CUDA(c, cudaMemcpyAsync(b + 8 * N, mem, 8 * N, cudaMemcpyHostToDevice, c->stream));
        if (gpu) GP_CUDA(c, cudaMemcpyAsync(b + 16 * N, gpu, 8 * N, cudaMemcpyHostToDevice, c->stream));
        else GP_CUDA(c, cudaMemsetAsync(b + 16 * N, 0, 8 * N, c->stream));
    }
    GP_CUDA(c, cudaStreamSynchronize(c->stream));
    c->have_sched = true;
    c->have_eff_sched = true;
    return GP_OK;
}

// ---- staging shared by the zone entry points ------------------------------------------------------------------------
// the arrays a non-empty batch of a zone entry point needs
static bool has_zone_arrays(const gp_apps* a, const gp_zone_results* out) {
    return a->drv_cpu_milli && a->drv_mem_bytes && a->exe_cpu_milli && a->exe_mem_bytes && a->exe_count && out->zone && out->driver_node;
}

// The six int64 quantity columns (6 x n_apps from o_in; absent gpu columns stay NULL = 0 in `six`), exe_count to o_cnt
// and the ExecutorNodes offsets `off` to o_off
static gp_status upload_app_columns(gp_ctx* c, const gp_apps* a, const int64_t* off, char* b, size_t o_in, size_t o_cnt, size_t o_off,
                                    cudaStream_t st, SixCols* six) {
    const size_t q = (size_t)a->n_apps;
    const int64_t* hc[6] = {a->drv_cpu_milli, a->drv_mem_bytes, a->drv_gpu, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu};
    *six = SixCols{};
    for (int k = 0; k < 6; ++k) {
        if (!hc[k]) continue;
        int64_t* d = reinterpret_cast<int64_t*>(b + o_in) + q * (size_t)k;
        GP_CUDA(c, cudaMemcpyAsync(d, hc[k], 8 * q, cudaMemcpyHostToDevice, st));
        six->p[k] = d;
    }
    GP_CUDA(c, cudaMemcpyAsync(b + o_cnt, a->exe_count, 4 * q, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(b + o_off, off, 8 * (q + 1), cudaMemcpyHostToDevice, st));
    return GP_OK;
}

// az-aware-tightly-pack: upload the undivided orders and build the fallback's gather view of them (gp_build_fallback_view).
// on_device: az's orders are device arrays (gp_prepare_cluster_zones' held orders) and are read in place.
static gp_status stage_fallback_view(gp_ctx* c, const gp_az_orders* az, bool on_device, cudaStream_t st, GatherSlots* fb) {
    const size_t ne = (size_t)az->n_exec, nd = (size_t)az->n_drv;
    Arena ar{c->fbview};
    const size_t o_eord = ar.take(on_device ? 0 : 4 * ne), o_dord = ar.take(on_device ? 0 : 4 * nd), o_npos = ar.take(4 * (size_t)c->n_nodes),
                 o_fbe = ar.take(4 * ne), o_fbd = ar.take(4 * nd), o_fbp = ar.take(4 * nd);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    const int32_t* eord = on_device ? az->exec_order : (const int32_t*)(b + o_eord);
    const int32_t* dord = on_device ? az->drv_order : (const int32_t*)(b + o_dord);
    if (!on_device && ne) GP_CUDA(c, cudaMemcpyAsync(b + o_eord, az->exec_order, 4 * ne, cudaMemcpyHostToDevice, st));
    if (!on_device && nd) GP_CUDA(c, cudaMemcpyAsync(b + o_dord, az->drv_order, 4 * nd, cudaMemcpyHostToDevice, st));
    gp_build_fallback_view<<<1, 1024, 0, st>>>(c->n_nodes, (int32_t)ne, (int32_t)nd, eord, dord,
                                               c->node_slot.as<int32_t>(), (int32_t*)(b + o_npos), (int32_t*)(b + o_fbe), (int32_t*)(b + o_fbd),
                                               (int32_t*)(b + o_fbp));
    c->last.kernel_launches += 1;
    *fb = GatherSlots{(const int32_t*)(b + o_fbe), (const int32_t*)(b + o_fbd), (const int32_t*)(b + o_fbp), (int32_t)ne, (int32_t)nd};
    return GP_OK;
}

// zone / driver / ExecutorNodes (T entries) / averages to the host, one synchronise, then the kernels' validation errors
static gp_status finish_zone_results(gp_ctx* c, gp_zone_results* out, const int32_t* zone, const int32_t* drv, const int32_t* exe,
                                     const double* avg, size_t q, size_t T, cudaStream_t st) {
    GP_CUDA(c, cudaMemcpyAsync(out->zone, zone, 4 * q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(out->driver_node, drv, 4 * q, cudaMemcpyDeviceToHost, st));
    if (T) GP_CUDA(c, cudaMemcpyAsync(out->executor_nodes, exe, 4 * T, cudaMemcpyDeviceToHost, st));
    if (out->avg_efficiency) GP_CUDA(c, cudaMemcpyAsync(out->avg_efficiency, avg, 32 * q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return host_error(c);
}

// Independent zone packs of a batch, shared by gp_pack_batch_zones (the zones are every instance group, no fallback) and
// gp_pack_batch_az_aware (zones 0..Z-1 with tightly-pack, plus the undivided orders `az` of the fallback, already
// validated; az_dev: they are device arrays).  Argument checks common to both are here.
static gp_status batch_zones_run(gp_ctx* c, const gp_apps* a, gp_algo algo, int32_t Z, const gp_az_orders* az, bool az_dev,
                                 gp_zone_results* out, const char* who) {
    const std::string w(who);
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    if (!has_zone_arrays(a, out)) return fail(c, GP_ERR_INVALID, w + ": missing app/result arrays");
    if ((int64_t)Q * Z > 0x7fffffffLL) return fail(c, GP_ERR_INVALID, w + ": n_apps x zones too large");
    const int64_t* off = a->exec_out_off;
    if (!off) {
        c->host_off.resize((size_t)Q + 1);
        int64_t acc = 0;
        for (int32_t i = 0; i < Q; ++i) { c->host_off[(size_t)i] = acc; acc += a->exe_count[i] > 0 ? a->exe_count[i] : 0; }
        c->host_off[(size_t)Q] = acc;
        off = c->host_off.data();
    }
    const int64_t total = off[Q];
    if (total < 0 || total > out->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, w + ": executor_nodes_cap too small");
    if (total > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, w + ": executor_nodes is NULL");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, R = q * (size_t)Z, T = (size_t)total;
    Arena ar{c->zonebuf};
    const size_t o_in = ar.take(48 * q), o_cnt = ar.take(4 * q), o_off = ar.take(8 * (q + 1)), o_rows = ar.take(48 * R), o_rcnt = ar.take(4 * R),
                 o_rgrp = ar.take(4 * R), o_roff = ar.take(8 * (R + 1)), o_rdrv = ar.take(4 * R), o_rexe = ar.take(4 * ((size_t)Z * T + 1)),
                 o_zone = ar.take(4 * q), o_drv = ar.take(4 * q), o_exe = ar.take(4 * (T + 1)), o_avg = ar.take(32 * q);
    // az-aware: the fallback's PrepApp records and list
    const size_t QF = az ? q : 0;
    const size_t o_prep = ar.take(sizeof(PrepApp) * QF), o_list = ar.take(4 * QF);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    SixCols six;
    gp_status s = upload_app_columns(c, a, off, b, o_in, o_cnt, o_off, st, &six);
    if (s != GP_OK) return s;
    const int TH = 256;
    // the efficiencies read the availability in node-table order: refresh that copy from the slots (a FIFO batch may
    // have charged them since gp_set_snapshot)
    if (c->n_slots > 0)
        gp_scatter_slots<<<(c->n_slots + TH - 1) / TH, TH, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), c->sgpu.as<int64_t>(), c->slot_node.as<int32_t>(),
                                                                   c->node_cpu.as<int64_t>(), c->node_mem.as<int64_t>(), c->node_gpu.as<int64_t>());
    gp_zone_expand<<<(unsigned)((R + 1 + TH - 1) / TH), TH, 0, st>>>(Q, Z, six, (const int32_t*)(b + o_cnt), (const int64_t*)(b + o_off),
                                                                      (int64_t*)(b + o_rows), (int32_t*)(b + o_rcnt), (int32_t*)(b + o_rgrp), (int64_t*)(b + o_roff));
    int2* scratch = nullptr;
    s = pack_begin(c, (int32_t)R, algo, GP_MODE_INDEPENDENT, (int64_t)Z * total, false, &scratch, st);
    if (s != GP_OK) return s;
    DevApps dv{};
    for (int k = 0; k < 6; ++k) dv.cols.q[k] = b + o_rows + 8 * R * (size_t)k;
    dv.cols.count = (const int32_t*)(b + o_rcnt); dv.cols.group = (const int32_t*)(b + o_rgrp); dv.cols.off = (const int64_t*)(b + o_roff);
    dv.cols.bits = 64; dv.cols.mem_shift = 0; dv.skip = nullptr; dv.n = (int32_t)R;
    DevResults dr{(int32_t*)(b + o_rdrv), b + o_rexe, (int64_t)Z * total, 32};
    s = pack_device_range(c, dv, 0, (int32_t)R, 0, algo, GP_MODE_INDEPENDENT, dr, scratch, st, 0);
    if (s != GP_OK) return s;
    c->ev_chunks = 1;
    ZoneChooseIn zi{};
    const size_t N = (size_t)c->n_nodes;
    zi.avail[0] = c->node_cpu.as<long long>(); zi.avail[1] = c->node_mem.as<long long>(); zi.avail[2] = c->node_gpu.as<long long>();
    zi.sched[0] = c->sched.as<long long>(); zi.sched[1] = c->sched.as<long long>() + N; zi.sched[2] = c->sched.as<long long>() + 2 * N;
    for (int k = 0; k < 3; ++k) { zi.drv[k] = six.p[k]; zi.exe[k] = six.p[3 + k]; }
    zi.count = (const int32_t*)(b + o_cnt); zi.out_off = (const int64_t*)(b + o_off);
    zi.row_driver = (const int32_t*)(b + o_rdrv); zi.row_exec = (const int32_t*)(b + o_rexe);
    zi.n_apps = Q; zi.n_zones = Z; zi.executors_reserved = algo == GP_TIGHTLY_PACK ? 1 : 0;
    gp_zone_choose<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(zi, (int32_t*)(b + o_zone), (int32_t*)(b + o_drv), (int32_t*)(b + o_exe),
                                                                       out->avg_efficiency ? (double*)(b + o_avg) : nullptr);
    GP_CUDA(c, cudaGetLastError());
    c->last.kernel_launches += 2;
    if (az) {
        // the applications no zone won: SparkBinPack(tightlyPackExecutors) over the undivided orders, still on the device
        // (az_aware_pack_tightly.go:33-37).  The list length and the fallback's claim counter are zeroed by pack_begin;
        // stats [2..3] restart so that scan_path_apps / _nodes count the fallback alone.
        DevStatus* ds = c->status();
        unsigned long long* d_stats = ds->head.stats;
        GP_CUDA(c, cudaMemsetAsync(d_stats + 2, 0, 16, st));
        int32_t* listed = (int32_t*)(b + o_list);
        gp_az_fallback_list<<<(unsigned)((q + TH - 1) / TH), TH, 0, st>>>(Q, (const int32_t*)(b + o_zone), listed, &ds->az_listed);
        AppColumns cols{};
        for (int k = 0; k < 6; ++k) cols.q[k] = six.p[k];
        cols.count = (const int32_t*)(b + o_cnt); cols.group = nullptr; cols.off = (const int64_t*)(b + o_off); cols.bits = 64; cols.mem_shift = 0;
        PrepApp* prep = (PrepApp*)(b + o_prep);
        gp_prep_apps<<<(Q + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, st>>>(
            Q, cols, nullptr, c->n_groups, total, c->snap_flags.as<SnapMeta>(), nullptr, prep, &ds->head.err, &c->host_status()->err_word);
        GatherSlots fb;
        s = stage_fallback_view(c, az, az_dev, st, &fb);
        if (s != GP_OK) return s;
        int& per_sm = c->az_fallback_ctas_per_sm;
        if (per_sm == 0) {
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gp_pack_az_fallback, kAzFallbackThreads, 0);
            if (per_sm < 1) per_sm = 1;
        }
        int64_t blocks = ((int64_t)Q * 32 + kAzFallbackThreads - 1) / kAzFallbackThreads;   // the list holds at most Q
        if (blocks > (int64_t)c->sm_count * per_sm) blocks = (int64_t)c->sm_count * per_sm;
        gp_pack_az_fallback<<<(unsigned)blocks, kAzFallbackThreads, 0, st>>>(make_snapshot(c), prep, listed, &ds->az_listed, fb, (int32_t*)(b + o_drv),
                                                                            (int32_t*)(b + o_exe), d_stats, &ds->az_claim);
        GP_CUDA(c, cudaGetLastError());
        c->last.kernel_launches += 3;
    }
    return finish_zone_results(c, out, (const int32_t*)(b + o_zone), (const int32_t*)(b + o_drv), (const int32_t*)(b + o_exe),
                               (const double*)(b + o_avg), q, T, st);
}

gp_status gp_pack_batch_zones(gp_ctx* c, const gp_apps* a, gp_algo algo, gp_zone_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_pack_batch_zones: gp_set_snapshot first");
    if (!c->have_sched) return fail(c, GP_ERR_INVALID, "gp_pack_batch_zones: gp_set_schedulable first (the efficiencies need SchedulableResources)");
    if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, "gp_pack_batch_zones: NULL apps/results");
    if (algo != GP_TIGHTLY_PACK && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, "gp_pack_batch_zones: the single-AZ packers are tightly-pack and minimal-fragmentation (single_az_pack_tightly.go, single_az_minimal_fragmentation.go)");
    return batch_zones_run(c, a, algo, c->n_groups, nullptr, false, out, "gp_pack_batch_zones");
}

// ---- reservation table + device-resident snapshot upkeep (gangpack_zones.cuh) -------------------------------------------
static gp_status refresh_views(gp_ctx* c, cudaStream_t st) {
    const int T = 256;
    if (c->n_slots <= 0) return GP_OK;
    SnapMeta* meta = c->snap_flags.as<SnapMeta>();
    gp_refresh_meta<<<(c->n_slots + T - 1) / T, T, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), c->sgpu.as<long long>(), c->slot_node.as<int32_t>(),
                                                           &meta->flags, meta->max_avail);
    gp_fill_pair32<<<(c->n_slots + T) / T, T, 0, st>>>(c->n_slots, c->pair.as<longlong2>(), meta, c->pair32.as<uint2>());
    GP_CUDA(c, cudaGetLastError());
    return GP_OK;
}

// The undivided orders of az-aware-tightly-pack against the snapshot gp_set_snapshot laid out, in O(N): every entry a node
// of the snapshot in that role, once; every zone group's order = the undivided order restricted to that group's nodes
// (the fallback and the zone packs must see the same priorities).  o->n_zones is already within 0..n_groups.
static gp_status check_az_orders(gp_ctx* c, const gp_az_orders* o, const char* who) {
    const std::string w(who);
    if (!c->host_layout)
        return fail(c, GP_ERR_INVALID, w + ": the snapshot must be laid out by gp_set_snapshot (after gp_set_snapshot_device / "
                                           "gp_prepare_cluster there is no host copy of the layout to check the undivided orders against)");
    if (o->n_exec != c->n_exec || o->n_drv != c->n_drv)
        return fail(c, GP_ERR_INVALID, w + ": order lengths must equal the snapshot's exec_off[n_groups] / drv_off[n_groups]");
    if ((o->n_exec > 0 && !o->exec_order) || (o->n_drv > 0 && !o->drv_order))
        return fail(c, GP_ERR_INVALID, w + ": order arrays missing");
    const int32_t Z = o->n_zones;
    const uint32_t N = (uint32_t)c->n_nodes;
    const int32_t* owner = c->v_owner.data();
    const int32_t* pos = c->v_pos.data();
    for (int role = 0; role < 2; ++role) {
        const int32_t n = role == 0 ? o->n_exec : o->n_drv;
        const int32_t* ord = role == 0 ? o->exec_order : o->drv_order;
        const char* name = role == 0 ? "exec_order" : "drv_order";
        std::vector<uint8_t>& seen = role == 0 ? c->v_seen_e : c->v_seen_d;
        seen.assign((size_t)N, 0);
        std::vector<int32_t>& next = c->v_zone_next;     // next expected position in each zone group's order
        next.assign((size_t)Z, 0);
        for (int32_t i = 0; i < n; ++i) {
            const uint32_t v = (uint32_t)ord[i];
            if (v >= N) return fail(c, GP_ERR_INVALID, w + ": " + name + " entry out of range");
            if (seen[v]) return fail(c, GP_ERR_INVALID, w + ": " + name + " lists a node twice");
            seen[v] = 1;
            const int32_t ow = owner[v];
            if (ow < 0 || !(ow & (1 << role)))
                return fail(c, GP_ERR_INVALID, w + ": " + name + " lists a node the snapshot does not list as " +
                                                   (role == 0 ? "an executor" : "a driver") + " candidate");
            const int32_t g = ow >> 2;
            if (g < Z && pos[(size_t)role * N + v] != next[(size_t)g]++)
                return fail(c, GP_ERR_INVALID, w + ": zone group " + std::to_string(g) + "'s " +
                                                   (role == 0 ? "executor" : "driver") + " order is not " + name + " restricted to its nodes");
        }
    }
    return GP_OK;
}

// The az-aware entries' NULL arguments.  orders == NULL stands for the undivided orders and n_zones gp_prepare_cluster_zones
// (GP_LAYOUT_AZ_AWARE) left on the device -- *o then points at them; after any other snapshot it is refused.
static gp_status held_az_orders(gp_ctx* c, const gp_apps* a, const gp_zone_results* out, const gp_az_orders** o, const char* who) {
    const std::string w(who);
    if (!*o && c->zone_kind == GP_LAYOUT_SINGLE_AZ)
        return fail(c, GP_ERR_INVALID, w + ": orders == NULL needs a gp_prepare_cluster_zones(GP_LAYOUT_AZ_AWARE) snapshot; this one is "
                                           "GP_LAYOUT_SINGLE_AZ (no trailing group, no undivided orders)");
    if (!a || !out || (!*o && c->zone_kind != GP_LAYOUT_AZ_AWARE) || a->n_apps < 0) return fail(c, GP_ERR_INVALID, w + ": NULL apps/orders/results");
    if (!*o) *o = &c->zone_orders;
    return GP_OK;
}

// The FIFO loop over zones in one launch (gangpack_zonefifo.cuh), shared by gp_pack_fifo_zones (kind = 0 tightly-pack,
// 2 minimal-fragmentation; the zones are every instance group) and gp_pack_fifo_az_aware (kind = kZoneAzAware; zones
// 0..Z-1, plus the undivided orders `az` of the fallback, already validated; az_dev: they are device arrays).  Argument
// checks common to both are here.
static gp_status fifo_zones_run(gp_ctx* c, const gp_apps* a, int kind, gp_mode mode, int32_t Z, const gp_az_orders* az, bool az_dev,
                                gp_zone_results* out, const char* who) {
    const std::string w(who);
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    if (!has_zone_arrays(a, out)) return fail(c, GP_ERR_INVALID, w + ": missing app/result arrays");
    std::vector<int64_t>& hoff = c->host_off;
    hoff.resize((size_t)Q + 1);
    int64_t acc = 0, pitch = 1;
    for (int32_t i = 0; i < Q; ++i) {
        const int64_t k = a->exe_count[i] > 0 ? a->exe_count[i] : 0;
        hoff[(size_t)i] = acc; acc += k;
        if (k > pitch) pitch = k;
    }
    hoff[(size_t)Q] = acc;
    if (a->exec_out_off)
        for (int32_t i = 0; i <= Q; ++i)
            if (a->exec_out_off[i] != hoff[(size_t)i]) return fail(c, GP_ERR_INVALID, w + ": exec_out_off must be the prefix sum of exe_count (or NULL)");
    const int64_t total = acc;
    if (total > out->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, w + ": executor_nodes_cap too small");
    if (total > 0 && !out->executor_nodes) return fail(c, GP_ERR_INVALID, w + ": executor_nodes is NULL");
    pitch = (pitch + 3) & ~(int64_t)3;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const bool azk = kind == kZoneAzAware;
    const size_t q = (size_t)Q, T = (size_t)total, RP = (size_t)(Z + (azk ? 1 : 0)) * (size_t)pitch;   // az-aware: row Z = fallback
    Arena ar{c->zonebuf};
    const size_t o_in = ar.take(48 * q), o_cnt = ar.take(4 * q), o_off = ar.take(8 * (q + 1)), o_skip = ar.take(q), o_rexe = ar.take(4 * RP),
                 o_rlist = ar.take(kind == GP_MINIMAL_FRAGMENTATION ? 8 * RP : 0), o_zone = ar.take(4 * q), o_drv = ar.take(4 * q),
                 o_exe = ar.take(4 * (T + 1)), o_avg = ar.take(32 * q);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    int2* unused = nullptr;
    gp_status s = pack_begin(c, Q, GP_TIGHTLY_PACK, mode, total, false, &unused, st);
    if (s != GP_OK) return s;
    SixCols six;
    s = upload_app_columns(c, a, hoff.data(), b, o_in, o_cnt, o_off, st, &six);
    if (s != GP_OK) return s;
    if (a->skip_if_no_fit) GP_CUDA(c, cudaMemcpyAsync(b + o_skip, a->skip_if_no_fit, q, cudaMemcpyHostToDevice, st));
    AppColumns cols{};
    for (int k = 0; k < 6; ++k) cols.q[k] = six.p[k];
    cols.count = (const int32_t*)(b + o_cnt); cols.group = nullptr; cols.off = (const int64_t*)(b + o_off); cols.bits = 64; cols.mem_shift = 0;
    DevStatus* ds = c->status();
    unsigned long long* d_stats = ds->head.stats;
    PrepApp* prep = c->prep.as<PrepApp>();
    gp_prep_apps<<<(Q + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, st>>>(
        Q, cols, a->skip_if_no_fit ? (const uint8_t*)(b + o_skip) : nullptr, c->n_groups, total, c->snap_flags.as<SnapMeta>(), nullptr, prep,
        &ds->head.err, &c->host_status()->err_word);
    Snapshot snap = make_snapshot(c);
    ZoneFifoIn zi{};
    const size_t N = (size_t)c->n_nodes;
    zi.sched[0] = c->sched.as<long long>(); zi.sched[1] = c->sched.as<long long>() + N; zi.sched[2] = c->sched.as<long long>() + 2 * N;
    zi.node_slot = c->node_slot.as<int32_t>();
    zi.row_exec = (int32_t*)(b + o_rexe);
    zi.row_list = kind == GP_MINIMAL_FRAGMENTATION ? (int2*)(b + o_rlist) : nullptr;
    zi.row_pitch = pitch; zi.n_apps = Q; zi.n_zones = Z;
    double* avg = out->avg_efficiency ? (double*)(b + o_avg) : nullptr;
    int32_t* zo = (int32_t*)(b + o_zone); int32_t* dq = (int32_t*)(b + o_drv); int32_t* eo = (int32_t*)(b + o_exe);
    GatherSlots fb{};
    if (azk) {
        s = stage_fallback_view(c, az, az_dev, st, &fb);
        if (s != GP_OK) return s;
    }
    if (kind == GP_TIGHTLY_PACK) {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<0, 1><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
        else gp_pack_fifo_zones_cta<0, 2><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
    } else if (kind == GP_MINIMAL_FRAGMENTATION) {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<2, 1><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
        else gp_pack_fifo_zones_cta<2, 2><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats);
    } else {
        if (mode == GP_MODE_FIFO_REFERENCE) gp_pack_fifo_zones_cta<kZoneAzAware, 1><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats, fb);
        else gp_pack_fifo_zones_cta<kZoneAzAware, 2><<<1, kZoneFifoThreads, 0, st>>>(snap, prep, zi, zo, dq, eo, avg, d_stats, fb);
    }
    GP_CUDA(c, cudaGetLastError());
    c->last.kernel_launches += 2;
    s = refresh_views(c, st);                          // the compact view follows the charged slots
    if (s != GP_OK) return s;
    return finish_zone_results(c, out, zo, dq, eo, avg, q, T, st);
}

// the FIFO loop with a single-AZ packer in one launch
gp_status gp_pack_fifo_zones(gp_ctx* c, const gp_apps* a, gp_algo algo, gp_mode mode, gp_zone_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_pack_fifo_zones: gp_set_snapshot first");
    if (!c->have_sched) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: gp_set_schedulable first (the efficiencies need SchedulableResources)");
    if (!a || !out || a->n_apps < 0) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: NULL apps/results");
    if (algo != GP_TIGHTLY_PACK && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: the single-AZ packers are tightly-pack and minimal-fragmentation");
    if (mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: mode must be one of the FIFO modes (independent decisions: gp_pack_batch_zones)");
    const int32_t Z = c->n_groups;
    if (Z > kZoneFifoMaxZones) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_zones: more than 64 zones");
    return fifo_zones_run(c, a, (int)algo, mode, Z, nullptr, false, out, "gp_pack_fifo_zones");
}

// the FIFO loop with az-aware-tightly-pack in one launch: the zone packs plus the undivided fallback on the device
gp_status gp_pack_fifo_az_aware(gp_ctx* c, const gp_apps* a, gp_mode mode, const gp_az_orders* o, gp_zone_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_pack_fifo_az_aware: gp_set_snapshot first");
    if (mode != GP_MODE_FIFO_REFERENCE && mode != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: mode must be one of the FIFO modes (independent decisions: gp_pack_batch_zones, "
                                       "then gp_pack_batch over the undivided orders)");
    if (!c->have_sched) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: gp_set_schedulable first (the efficiencies need SchedulableResources)");
    gp_status s = held_az_orders(c, a, out, &o, "gp_pack_fifo_az_aware");
    if (s != GP_OK) return s;
    const bool held = o == &c->zone_orders;
    const int32_t Z = o->n_zones;
    if (Z < 0 || Z > kZoneFifoMaxZones) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: n_zones must be 0..64");
    if (Z > c->n_groups) return fail(c, GP_ERR_INVALID, "gp_pack_fifo_az_aware: n_zones exceeds the snapshot's instance groups");
    if (!held) s = check_az_orders(c, o, "gp_pack_fifo_az_aware");
    if (s != GP_OK) return s;
    return fifo_zones_run(c, a, kZoneAzAware, mode, Z, o, held, out, "gp_pack_fifo_az_aware");
}

// az-aware-tightly-pack for a batch of independent decisions: the zone packs, the zone choice and the undivided fallback
// on the device, one stream synchronise
gp_status gp_pack_batch_az_aware(gp_ctx* c, const gp_apps* a, const gp_az_orders* o, gp_zone_results* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_pack_batch_az_aware: gp_set_snapshot first");
    if (!c->have_sched) return fail(c, GP_ERR_INVALID, "gp_pack_batch_az_aware: gp_set_schedulable first (the efficiencies need SchedulableResources)");
    gp_status s = held_az_orders(c, a, out, &o, "gp_pack_batch_az_aware");
    if (s != GP_OK) return s;
    const bool held = o == &c->zone_orders;
    const int32_t Z = o->n_zones;
    if (Z < 0) return fail(c, GP_ERR_INVALID, "gp_pack_batch_az_aware: n_zones is negative");
    if (Z > c->n_groups) return fail(c, GP_ERR_INVALID, "gp_pack_batch_az_aware: n_zones exceeds the snapshot's instance groups");
    if (!held) s = check_az_orders(c, o, "gp_pack_batch_az_aware");
    if (s != GP_OK) return s;
    return batch_zones_run(c, a, GP_TIGHTLY_PACK, Z, o, held, out, "gp_pack_batch_az_aware");
}

gp_status gp_reserve_placements(gp_ctx* c, const gp_apps* a, const gp_results* placed, int32_t subtract, gp_reservation_table* out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_reserve_placements: gp_set_snapshot first");
    if (!a || !placed || a->n_apps < 0 || (!out && !subtract)) return fail(c, GP_ERR_INVALID, "gp_reserve_placements: NULL arguments");
    const int32_t Q = a->n_apps;
    if (out) out->n_rows = 0;
    if (Q == 0) return GP_OK;
    if (!a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !placed->driver_node)
        return fail(c, GP_ERR_INVALID, "gp_reserve_placements: missing app/result arrays");
    // host pass: offsets, rows per placed application, index validation
    std::vector<int64_t>& off = c->host_off;
    off.resize(2 * ((size_t)Q + 1));
    int64_t* roff = off.data() + Q + 1;
    int64_t acc = 0, rows = 0;
    for (int32_t i = 0; i < Q; ++i) {
        const int64_t k = a->exe_count[i] > 0 ? a->exe_count[i] : 0;
        off[(size_t)i] = a->exec_out_off ? a->exec_out_off[i] : acc;
        acc += k;
        roff[i] = rows;
        const int32_t d = placed->driver_node[i];
        if (d >= c->n_nodes) return fail(c, GP_ERR_INVALID, "gp_reserve_placements: driver_node out of range");
        if (d >= 0) {
            if (k > 0 && !placed->executor_nodes) return fail(c, GP_ERR_INVALID, "gp_reserve_placements: executor_nodes is NULL");
            if (off[(size_t)i] < 0 || off[(size_t)i] + k > placed->executor_nodes_cap) return fail(c, GP_ERR_CAPACITY, "gp_reserve_placements: offsets exceed executor_nodes_cap");
            for (int64_t t = 0; t < k; ++t) {
                const int32_t n = placed->executor_nodes[off[(size_t)i] + t];
                if (n < 0 || n >= c->n_nodes) return fail(c, GP_ERR_INVALID, "gp_reserve_placements: executor node out of range");
            }
            rows += 1 + k;
        }
    }
    off[(size_t)Q] = a->exec_out_off ? a->exec_out_off[Q] : acc;
    roff[Q] = rows;
    const int64_t total = placed->executor_nodes_cap < off[(size_t)Q] ? placed->executor_nodes_cap : off[(size_t)Q];
    if (out && rows > out->rows_cap) return fail(c, GP_ERR_CAPACITY, "gp_reserve_placements: rows_cap too small");
    if (out && rows > 0 && (!out->app || !out->slot || !out->node || !out->cpu_milli || !out->mem_bytes))
        return fail(c, GP_ERR_INVALID, "gp_reserve_placements: missing table arrays");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, T = (size_t)(total > 0 ? total : 0), R = (size_t)rows;
    Arena ar{c->zonebuf};
    const size_t o_in = ar.take(48 * q), o_cnt = ar.take(4 * q), o_off = ar.take(8 * (q + 1)), o_roff = ar.take(8 * (q + 1)), o_drv = ar.take(4 * q),
                 o_exe = ar.take(4 * (T + 1)), o_ra = ar.take(4 * (R + 1)), o_rs = ar.take(4 * (R + 1)), o_rn = ar.take(4 * (R + 1)),
                 o_rc = ar.take(8 * (R + 1)), o_rm = ar.take(8 * (R + 1)), o_rg = ar.take(8 * (R + 1));
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    ReserveIn ri{};
    gp_status s = upload_app_columns(c, a, off.data(), b, o_in, o_cnt, o_off, st, &ri.cols);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaMemcpyAsync(b + o_roff, roff, 8 * (q + 1), cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(b + o_drv, placed->driver_node, 4 * q, cudaMemcpyHostToDevice, st));
    if (T) GP_CUDA(c, cudaMemcpyAsync(b + o_exe, placed->executor_nodes, 4 * T, cudaMemcpyHostToDevice, st));
    ri.count = (const int32_t*)(b + o_cnt); ri.off = (const int64_t*)(b + o_off); ri.row_off = (const int64_t*)(b + o_roff);
    ri.driver = (const int32_t*)(b + o_drv); ri.exec = (const int32_t*)(b + o_exe); ri.n_apps = Q; ri.subtract = subtract ? 1 : 0;
    ReserveOut ro{(int32_t*)(b + o_ra), (int32_t*)(b + o_rs), (int32_t*)(b + o_rn), (long long*)(b + o_rc), (long long*)(b + o_rm), (long long*)(b + o_rg)};
    const int TH = 256;
    gp_reserve_rows<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(ri, ro, c->node_slot.as<int32_t>(), c->pair.as<longlong2>(), c->sgpu.as<long long>(),
                                                                        c->node_cpu.as<long long>(), c->node_mem.as<long long>(), c->node_gpu.as<long long>());
    GP_CUDA(c, cudaGetLastError());
    if (subtract) { s = refresh_views(c, st); if (s != GP_OK) return s; }
    if (out && R) {
        GP_CUDA(c, cudaMemcpyAsync(out->app, ro.app, 4 * R, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(out->slot, ro.slot, 4 * R, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(out->node, ro.node, 4 * R, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(out->cpu_milli, ro.cpu, 8 * R, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(out->mem_bytes, ro.mem, 8 * R, cudaMemcpyDeviceToHost, st));
        if (out->gpu) GP_CUDA(c, cudaMemcpyAsync(out->gpu, ro.gpu, 8 * R, cudaMemcpyDeviceToHost, st));
    }
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (out) out->n_rows = rows;
    return GP_OK;
}

gp_status gp_apply_usage_delta(gp_ctx* c, int64_t n_rows, const int32_t* node, const int64_t* cpu, const int64_t* mem, const int64_t* gpu, int32_t sign) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_apply_usage_delta: gp_set_snapshot first");
    if (n_rows < 0 || (sign != 1 && sign != -1) || (n_rows > 0 && (!node || !cpu || !mem))) return fail(c, GP_ERR_INVALID, "gp_apply_usage_delta: bad arguments");
    if (n_rows == 0) return GP_OK;
    for (int64_t r = 0; r < n_rows; ++r) {
        const int64_t v[3] = {cpu[r], mem[r], gpu ? gpu[r] : 0};
        for (int64_t x : v) if (x >= kMaxQuantity || x <= -kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_apply_usage_delta: |quantity| >= 2^61");
    }
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t R = (size_t)n_rows;
    Arena ar{c->zonebuf};
    const size_t o_c = ar.take(8 * R), o_m = ar.take(8 * R), o_g = ar.take(8 * R), o_n = ar.take(4 * R);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    GP_CUDA(c, cudaMemcpyAsync(b + o_c, cpu, 8 * R, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(b + o_m, mem, 8 * R, cudaMemcpyHostToDevice, st));
    if (gpu) GP_CUDA(c, cudaMemcpyAsync(b + o_g, gpu, 8 * R, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(b + o_n, node, 4 * R, cudaMemcpyHostToDevice, st));
    const int TH = 256;
    gp_usage_delta<<<(unsigned)((R + TH - 1) / TH), TH, 0, st>>>(n_rows, (const int32_t*)(b + o_n), (const long long*)(b + o_c), (const long long*)(b + o_m),
                                                                  gpu ? (const long long*)(b + o_g) : nullptr, sign, c->n_nodes, c->node_slot.as<int32_t>(),
                                                                  c->pair.as<longlong2>(), c->sgpu.as<long long>(), c->node_cpu.as<long long>(),
                                                                  c->node_mem.as<long long>(), c->node_gpu.as<long long>());
    GP_CUDA(c, cudaGetLastError());
    gp_status s = refresh_views(c, st);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

// ---- computeAvgPackingEfficiencyForResult over the whole node table, exactly summed (gangpack_efficiency.cuh) ----------
gp_status gp_packing_efficiency(gp_ctx* c, const gp_apps* a, gp_algo algo, const gp_results* placed, gp_mode charged, double* avg_out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_packing_efficiency: no snapshot (gp_set_snapshot, gp_prepare_cluster or gp_prepare_cluster_zones first)");
    if (!c->have_eff_sched)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: no SchedulableResources (gp_set_schedulable, gp_prepare_cluster or gp_prepare_cluster_zones first)");
    if (!a || !placed || a->n_apps < 0) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: NULL apps/placed");
    if (algo != GP_TIGHTLY_PACK && algo != GP_DISTRIBUTE_EVENLY && algo != GP_MINIMAL_FRAGMENTATION)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: unknown algo");
    if (charged != GP_MODE_INDEPENDENT && charged != GP_MODE_FIFO_REFERENCE && charged != GP_MODE_FIFO_EXACT)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: unknown charged mode");
    if (charged != GP_MODE_INDEPENDENT && a->n_apps != 1)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: a FIFO charged mode adds back ONE application's usage: n_apps must be 1");
    const int32_t Q = a->n_apps;
    if (Q == 0) return GP_OK;
    if (!avg_out || !a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !placed->driver_node)
        return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: missing app/result arrays");
    // host pass over the placed rows: offsets, request domain, node indices (a caller-supplied placement need not be feasible)
    std::vector<int64_t>& off = c->host_off;
    off.resize((size_t)Q + 1);
    const int64_t* qc[6] = {a->drv_cpu_milli, a->drv_mem_bytes, a->drv_gpu, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu};
    int64_t acc = 0;
    for (int32_t i = 0; i < Q; ++i) {
        const int64_t k = a->exe_count[i] > 0 ? a->exe_count[i] : 0;
        off[(size_t)i] = a->exec_out_off ? a->exec_out_off[i] : acc;
        acc += k;
        const int32_t d = placed->driver_node[i];
        if (d >= c->n_nodes) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: driver_node out of range");
        if (d < 0) continue;
        for (const int64_t* col : qc) {
            if (!col) continue;
            if (col[i] < 0) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: negative request");
            if (col[i] >= kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_packing_efficiency: request >= 2^61");
        }
        if (k > 0 && !placed->executor_nodes) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: executor_nodes is NULL");
        if (off[(size_t)i] < 0 || off[(size_t)i] + k > placed->executor_nodes_cap)
            return fail(c, GP_ERR_CAPACITY, "gp_packing_efficiency: offsets exceed executor_nodes_cap");
        for (int64_t t = 0; t < k; ++t) {
            const int32_t n = placed->executor_nodes[off[(size_t)i] + t];
            if (n < 0 || n >= c->n_nodes) return fail(c, GP_ERR_INVALID, "gp_packing_efficiency: executor node out of range");
        }
    }
    off[(size_t)Q] = a->exec_out_off ? a->exec_out_off[Q] : acc;
    const int64_t total = placed->executor_nodes_cap < off[(size_t)Q] ? placed->executor_nodes_cap : off[(size_t)Q];
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t q = (size_t)Q, T = (size_t)(total > 0 ? total : 0), N = (size_t)c->n_nodes;
    const int TH = kEffThreads;
    const int n_part = (int)std::max<size_t>(1, std::min<size_t>((N + TH - 1) / TH, (size_t)c->sm_count * 4));
    Arena ar{c->zonebuf};
    const size_t o_in = ar.take(48 * q), o_cnt = ar.take(4 * q), o_off = ar.take(8 * (q + 1)), o_drv = ar.take(4 * q), o_exe = ar.take(4 * (T + 1)),
                 o_part = ar.take(sizeof(EffAcc) * (size_t)n_part), o_base = ar.take(sizeof(EffAcc)), o_avg = ar.take(32 * q), o_err = ar.take(4);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    EffRowsIn ri{};
    gp_status s = upload_app_columns(c, a, off.data(), b, o_in, o_cnt, o_off, st, &ri.cols);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaMemcpyAsync(b + o_drv, placed->driver_node, 4 * q, cudaMemcpyHostToDevice, st));
    if (T) GP_CUDA(c, cudaMemcpyAsync(b + o_exe, placed->executor_nodes, 4 * T, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_err, 0, 4, st));
    int* d_err = (int*)(b + o_err);
    EffBaseIn bi{};
    bi.av = SnapshotAvail{c->pair.as<longlong2>(), c->sgpu.as<long long>(), c->node_slot.as<int32_t>(), c->node_cpu.as<long long>(),
                      c->node_mem.as<long long>(), c->node_gpu.as<long long>()};
    bi.sched[0] = c->sched.as<long long>(); bi.sched[1] = c->sched.as<long long>() + N; bi.sched[2] = c->sched.as<long long>() + 2 * N;
    bi.n_nodes = c->n_nodes;
    EffAcc* base = (EffAcc*)(b + o_base);
    gp_eff_base<<<n_part, TH, 0, st>>>(bi, (EffAcc*)(b + o_part), d_err);
    gp_eff_finish<<<1, TH, 0, st>>>((const EffAcc*)(b + o_part), n_part, base);
    ri.av = bi.av;
    for (int k = 0; k < 3; ++k) ri.sched[k] = bi.sched[k];
    ri.count = (const int32_t*)(b + o_cnt); ri.off = (const int64_t*)(b + o_off);
    ri.driver = (const int32_t*)(b + o_drv); ri.exec = (const int32_t*)(b + o_exe); ri.base = base;
    ri.n_apps = Q; ri.n_nodes = c->n_nodes;
    ri.executors_reserved = algo == GP_MINIMAL_FRAGMENTATION ? 0 : 1;
    ri.charged = (int32_t)charged;
    gp_eff_rows<<<(unsigned)((q * 32 + TH - 1) / TH), TH, 0, st>>>(ri, (double*)(b + o_avg), d_err);
    GP_CUDA(c, cudaGetLastError());
    int herr = 0;
    GP_CUDA(c, cudaMemcpyAsync(avg_out, b + o_avg, 32 * q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (herr & kEffErrQuantity)
        return fail(c, GP_ERR_UNREPRESENTABLE, "gp_packing_efficiency: a per-node reserved amount is >= 2^61");
    if (herr & kEffErrRange)
        return fail(c, GP_ERR_UNREPRESENTABLE, "gp_packing_efficiency: an efficiency term outside the exact accumulator's range");
    return GP_OK;
}

// ---- node priority order (f1) and availability snapshot (f2): device stages + the entries built on them ----
}  // extern "C"

// Host checks shared by the entries below; `who` (the entry's name) prefixes every message.  The shape of a gp_usage_input:
// sizes non-negative, the allocatable columns for nodes, the reservation columns for rows.
static gp_status check_usage(gp_ctx* c, const gp_usage_input* in, const char* who) {
    if (!in || in->n_nodes < 0 || in->n_reservations < 0 || (in->n_nodes > 0 && (!in->alloc_cpu_milli || !in->alloc_mem_bytes)) ||
        (in->n_reservations > 0 && (!in->res_node || !in->res_cpu_milli || !in->res_mem_bytes)))
        return fail(c, GP_ERR_INVALID, std::string(who) + ": missing arrays or bad sizes");
    return GP_OK;
}

// The two id arrays of a gp_sort_input the kernels index with.
static gp_status check_sort_ids(gp_ctx* c, const gp_sort_input* in, const char* who) {
    const int32_t n = in->n_nodes;
    if (in->zone_id) for (int32_t i = 0; i < n; ++i)
        if (in->zone_id[i] < 0 || in->zone_id[i] >= in->n_zones) return fail(c, GP_ERR_INVALID, std::string(who) + ": zone_id out of range");
    if (in->name_rank) for (int32_t i = 0; i < n; ++i)
        if (in->name_rank[i] < 0 || in->name_rank[i] >= n) return fail(c, GP_ERR_INVALID, std::string(who) + ": name_rank out of range");
    return GP_OK;
}

// Executor requests (gpu optional): non-negative and inside the exact-int64 domain.
static gp_status check_requests(gp_ctx* c, int32_t q, const int64_t* cpu, const int64_t* mem, const int64_t* gpu, const char* who) {
    for (int32_t i = 0; i < q; ++i) {
        const int64_t v[3] = {cpu[i], mem[i], gpu ? gpu[i] : 0};
        for (int64_t x : v) {
            if (x < 0) return fail(c, GP_ERR_INVALID, std::string(who) + ": negative resource request");
            if (x >= kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, std::string(who) + ": quantity >= 2^61");
        }
    }
    return GP_OK;
}

// The host_off / host_nodes CSR of a gp_reschedule (host_off given): monotone from 0, node indices below n_nodes.
// *hosted = host_off[n_execs].
static gp_status check_hosting(gp_ctx* c, const gp_reschedule* in, int32_t n_nodes, int64_t* hosted, const char* who) {
    const std::string w(who);
    if (in->host_off[0] != 0) return fail(c, GP_ERR_INVALID, w + ": host_off must start at 0");
    for (int32_t i = 0; i < in->n_execs; ++i)
        if (in->host_off[i + 1] < in->host_off[i]) return fail(c, GP_ERR_INVALID, w + ": host_off not monotone");
    *hosted = in->host_off[in->n_execs];
    if (*hosted > 0 && !in->host_nodes) return fail(c, GP_ERR_INVALID, w + ": host_nodes missing");
    for (int64_t t = 0; t < *hosted; ++t)
        if (in->host_nodes[t] < 0 || in->host_nodes[t] >= n_nodes) return fail(c, GP_ERR_INVALID, w + ": host_nodes index out of range");
    return GP_OK;
}

// f2 stage: uploads the inputs, leaves avail[3][N] / sched[3][N] on the device (usagebuf).
// d_over (optional, [3]): the uploaded overhead columns, NULL where the caller gave none.
static gp_status stage_availability(gp_ctx* c, const gp_usage_input* in, cudaStream_t st, long long** d_avail, long long** d_sched,
                                    long long** d_resched = nullptr, const long long** d_over = nullptr) {
    const int32_t n = in->n_nodes;
    const size_t N = (size_t)n, R = (size_t)in->n_reservations;
    Arena ar{c->usagebuf};
    const size_t o_alloc = ar.take(24 * N), o_over = ar.take(24 * N), o_usage = ar.take(24 * N + 4 * N), o_avail = ar.take(24 * N),
                 o_sched = ar.take(24 * N), o_resched = ar.take(24 * N), o_rn = ar.take(4 * R), o_rc = ar.take(8 * R), o_rm = ar.take(8 * R),
                 o_rg = ar.take(8 * R);
    const size_t o_has = o_usage + 24 * N;      // zeroed together with the usage sums
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    GP_CUDA(c, ar.upload(o_alloc, in->alloc_cpu_milli, 8 * N, st));
    GP_CUDA(c, ar.upload(o_alloc + 8 * N, in->alloc_mem_bytes, 8 * N, st));
    if (in->alloc_gpu) GP_CUDA(c, ar.upload(o_alloc + 16 * N, in->alloc_gpu, 8 * N, st));
    if (in->overhead_cpu_milli) GP_CUDA(c, ar.upload(o_over, in->overhead_cpu_milli, 8 * N, st));
    if (in->overhead_mem_bytes) GP_CUDA(c, ar.upload(o_over + 8 * N, in->overhead_mem_bytes, 8 * N, st));
    if (in->overhead_gpu) GP_CUDA(c, ar.upload(o_over + 16 * N, in->overhead_gpu, 8 * N, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_usage, 0, 28 * N, st));
    const int T = 256;
    if (R) {
        GP_CUDA(c, ar.upload(o_rn, in->res_node, 4 * R, st));
        GP_CUDA(c, ar.upload(o_rc, in->res_cpu_milli, 8 * R, st));
        GP_CUDA(c, ar.upload(o_rm, in->res_mem_bytes, 8 * R, st));
        if (in->res_gpu) GP_CUDA(c, ar.upload(o_rg, in->res_gpu, 8 * R, st));
        gp_usage_scatter<<<(unsigned)((R + T - 1) / T), T, 0, st>>>((long long)R, (const int32_t*)(b + o_rn), (const long long*)(b + o_rc),
                                                                   (const long long*)(b + o_rm), in->res_gpu ? (const long long*)(b + o_rg) : nullptr,
                                                                   n, (unsigned long long*)(b + o_usage), d_resched ? (unsigned int*)(b + o_has) : nullptr);
    }
    const long long* al = (const long long*)(b + o_alloc);
    const long long* ov = (const long long*)(b + o_over);
    gp_availability<<<(n + T - 1) / T, T, 0, st>>>(n, al, al + N, in->alloc_gpu ? al + 2 * N : nullptr, in->overhead_cpu_milli ? ov : nullptr,
                                                   in->overhead_mem_bytes ? ov + N : nullptr, in->overhead_gpu ? ov + 2 * N : nullptr,
                                                   (const unsigned long long*)(b + o_usage), (long long*)(b + o_avail), (long long*)(b + o_sched),
                                                   (const unsigned int*)(b + o_has), d_resched ? (long long*)(b + o_resched) : nullptr);
    if (d_resched) *d_resched = (long long*)(b + o_resched);
    if (d_over) {
        d_over[0] = in->overhead_cpu_milli ? ov : nullptr;
        d_over[1] = in->overhead_mem_bytes ? ov + N : nullptr;
        d_over[2] = in->overhead_gpu ? ov + 2 * N : nullptr;
    }
    GP_CUDA(c, cudaGetLastError());
    *d_avail = (long long*)(b + o_avail);
    *d_sched = (long long*)(b + o_sched);
    return GP_OK;
}

struct SortStage { const int32_t* drv; const int32_t* exe; const int32_t* counts; const int32_t* zone; };

// Stable re-sort of list[0..*cnt) by rank[node] (-1 last): out[k] = the k-th node in (rank, position) order.  The label
// re-sort of PotentialNodes, and the zone partition of gp_prepare_cluster_zones.
static void launch_label_resort(int32_t n, const int32_t* cnt, const int32_t* list, const int32_t* rank, LabelKey* lk, LabelKey* lks,
                                int32_t* pos, int32_t* out, cudaStream_t st) {
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int ntile = (n + kSortTile - 1) / kSortTile;
    gp_label_keys<<<nb, T, 0, st>>>(cnt, list, rank, lk);
    gp_sort_tiles<LabelKey><<<ntile, kSortThreads, kSortTile * sizeof(LabelKey), st>>>(n, cnt, lk, lks);
    gp_rank_by_search<LabelKey><<<nb, T, 0, st>>>(n, cnt, lk, lks, pos);
    gp_label_scatter<<<nb, T, 0, st>>>(cnt, list, pos, out);
}

// f1 stage: d_cpu / d_mem / d_gpu are device arrays (NULL: uploaded from `in`; gpu optional); leaves the two orders,
// counts[3] = {#driver candidates, #executor candidates, #undefined ties} and the zone ids (NULL: one zone) on the device.
// The caller has run check_sort_ids.
static gp_status stage_sort(gp_ctx* c, const gp_sort_input* in, const long long* d_cpu, const long long* d_mem, const long long* d_gpu,
                            cudaStream_t st, SortStage* out) {
    const int32_t n = in->n_nodes;
    // one scratch block
    const size_t N = (size_t)n, Z = (size_t)in->n_zones;
    Arena ar{c->sortbuf};
    const size_t o_cpu = ar.take(8 * N), o_mem = ar.take(8 * N), o_gpu = ar.take(8 * N), o_keys = ar.take(sizeof(SortKey) * N),
                 o_sorted = ar.take(sizeof(SortKey) * N), o_tot = ar.take(16 * Z), o_zone = ar.take(4 * N), o_nr = ar.take(4 * N),
                 o_prio = ar.take(4 * Z), o_pos = ar.take(4 * N), o_order = ar.take(4 * N), o_drv = ar.take(4 * N), o_exe = ar.take(4 * N),
                 o_drv2 = ar.take(4 * N), o_exe2 = ar.take(4 * N), o_lrd = ar.take(4 * N), o_lre = ar.take(4 * N),
                 o_lk = ar.take(sizeof(LabelKey) * N), o_lks = ar.take(sizeof(LabelKey) * N), o_cnt = ar.take(16),
                 o_fc = ar.take(N), o_fu = ar.take(N), o_fr = ar.take(N);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    if (!d_cpu) { GP_CUDA(c, ar.upload(o_cpu, in->avail_cpu_milli, 8 * N, st)); d_cpu = (const long long*)(b + o_cpu); }
    if (!d_mem) { GP_CUDA(c, ar.upload(o_mem, in->avail_mem_bytes, 8 * N, st)); d_mem = (const long long*)(b + o_mem); }
    if (!d_gpu && in->avail_gpu) { GP_CUDA(c, ar.upload(o_gpu, in->avail_gpu, 8 * N, st)); d_gpu = (const long long*)(b + o_gpu); }
    const bool zoned = in->zone_id != nullptr && in->n_zones > 1;       // one zone: priority 0 for every node, nothing to total
    if (zoned) GP_CUDA(c, ar.upload(o_zone, in->zone_id, 4 * N, st));
    if (in->name_rank) GP_CUDA(c, ar.upload(o_nr, in->name_rank, 4 * N, st));
    if (in->is_driver_candidate) GP_CUDA(c, ar.upload(o_fc, in->is_driver_candidate, N, st));
    if (in->unschedulable) GP_CUDA(c, ar.upload(o_fu, in->unschedulable, N, st));
    if (in->ready) GP_CUDA(c, ar.upload(o_fr, in->ready, N, st));
    if (in->driver_label_rank) GP_CUDA(c, ar.upload(o_lrd, in->driver_label_rank, 4 * N, st));
    if (in->executor_label_rank) GP_CUDA(c, ar.upload(o_lre, in->executor_label_rank, 4 * N, st));
    if (zoned) GP_CUDA(c, cudaMemsetAsync(b + o_tot, 0, 16 * Z, st));
    if (!c->sort_attr_set) {
        GP_CUDA(c, cudaFuncSetAttribute(gp_sort_tiles<SortKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSortTile * sizeof(SortKey))));
        c->sort_attr_set = true;
    }
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int ntile = (n + kSortTile - 1) / kSortTile;
    SortKey* keys = (SortKey*)(b + o_keys);
    SortKey* sorted = (SortKey*)(b + o_sorted);
    int32_t* pos = (int32_t*)(b + o_pos);
    if (zoned) {
        gp_zone_totals<<<nb, T, 0, st>>>(n, d_cpu, d_mem, (const int32_t*)(b + o_zone), (unsigned long long*)(b + o_tot));
        gp_zone_priority<<<(in->n_zones + T - 1) / T, T, 0, st>>>(in->n_zones, (const unsigned long long*)(b + o_tot), (int32_t*)(b + o_prio));
    }
    gp_make_keys<<<nb, T, 0, st>>>(n, d_cpu, d_mem, zoned ? (const int32_t*)(b + o_zone) : nullptr, (const int32_t*)(b + o_prio),
                                   in->name_rank ? (const int32_t*)(b + o_nr) : nullptr, keys);
    gp_sort_tiles<SortKey><<<ntile, kSortThreads, kSortTile * sizeof(SortKey), st>>>(n, nullptr, keys, sorted);
    gp_rank_by_search<SortKey><<<nb, T, 0, st>>>(n, nullptr, keys, sorted, pos);
    gp_scatter_order<<<nb, T, 0, st>>>(n, pos, (int32_t*)(b + o_order));
    gp_split_candidates<<<1, 1024, 0, st>>>(n, (const int32_t*)(b + o_order), in->is_driver_candidate ? (const uint8_t*)(b + o_fc) : nullptr,
                                           in->unschedulable ? (const uint8_t*)(b + o_fu) : nullptr, in->ready ? (const uint8_t*)(b + o_fr) : nullptr,
                                           keys, d_gpu, (int32_t*)(b + o_drv), (int32_t*)(b + o_exe), (int32_t*)(b + o_cnt));
    out->drv = (const int32_t*)(b + o_drv);
    out->exe = (const int32_t*)(b + o_exe);
    out->counts = (const int32_t*)(b + o_cnt);
    out->zone = zoned ? (const int32_t*)(b + o_zone) : nullptr;
    auto label_sort = [&](const int32_t* cnt, const int32_t* list, size_t o_rank, size_t o_out) {
        launch_label_resort(n, cnt, list, (const int32_t*)(b + o_rank), (LabelKey*)(b + o_lk), (LabelKey*)(b + o_lks), pos,
                            (int32_t*)(b + o_out), st);
        return (const int32_t*)(b + o_out);
    };
    if (in->driver_label_rank) out->drv = label_sort(out->counts, out->drv, o_lrd, o_drv2);
    if (in->executor_label_rank) out->exe = label_sort(out->counts + 1, out->exe, o_lre, o_exe2);
    GP_CUDA(c, cudaGetLastError());
    return GP_OK;
}

// offsets of the single instance group from the device-resident candidate counts
__global__ void gp_offsets_from_counts(const int32_t* __restrict__ counts, int32_t* __restrict__ exec_off, int32_t* __restrict__ drv_off) {
    if (threadIdx.x == 0) { drv_off[0] = 0; drv_off[1] = counts[0]; exec_off[0] = 0; exec_off[1] = counts[1]; }
}

// gp_prepare_cluster and gp_prepare_cluster_zones up to their layout step: the checks both make, then reservations ->
// availability (d_avail / d_sched: [3][n_nodes]) -> priority orders on the context's stream.
static gp_status prepare_orders(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, const char* who,
                                long long** d_avail, long long** d_sched, SortStage* so) {
    gp_status s = check_usage(c, usage, who);
    if (s != GP_OK) return s;
    if (!sort || usage->n_nodes != sort->n_nodes || sort->n_zones < 1)
        return fail(c, GP_ERR_INVALID, std::string(who) + ": missing arrays or mismatched sizes");
    if (usage->n_nodes == 0) return fail(c, GP_ERR_INVALID, std::string(who) + ": empty node table");
    if ((s = check_sort_ids(c, sort, who)) != GP_OK) return s;
    GP_CUDA(c, cudaSetDevice(c->device));
    if ((s = stage_availability(c, usage, c->stream, d_avail, d_sched)) != GP_OK) return s;
    const size_t N = (size_t)usage->n_nodes;
    return stage_sort(c, sort, *d_avail, *d_avail + N, *d_avail + 2 * N, c->stream, so);
}

// gp_prepare_cluster and gp_prepare_cluster_zones after their layout step, which set dn's groups, offsets and orders: the
// node-table copy (gp_get_snapshot), the usual slot layout with n_nodes bounding both order lengths, SchedulableResources,
// and counts[3] of the sort read back (the caller synchronises).
static gp_status prepare_snapshot(gp_ctx* c, gp_nodes* dn, const long long* d_avail, const long long* d_sched, const SortStage& so,
                                  int32_t* counts) {
    cudaStream_t st = c->stream;
    const int32_t n = dn->n_nodes;
    const size_t N = (size_t)n, nb = sizeof(int64_t) * (N + 1);
    GP_CUDA(c, c->node_cpu.reserve(nb)); GP_CUDA(c, c->node_mem.reserve(nb)); GP_CUDA(c, c->node_gpu.reserve(nb));
    GP_CUDA(c, cudaMemcpyAsync(c->node_cpu.p, d_avail, 8 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(c->node_mem.p, d_avail + N, 8 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(c->node_gpu.p, d_avail + 2 * N, 8 * N, cudaMemcpyDeviceToDevice, st));
    dn->avail_cpu_milli = c->node_cpu.as<int64_t>(); dn->avail_mem_bytes = c->node_mem.as<int64_t>(); dn->avail_gpu = c->node_gpu.as<int64_t>();
    gp_status s = build_snapshot_device(c, dn, n, n, st);
    if (s != GP_OK) return s;
    GP_CUDA(c, c->sched.reserve(24 * (N + 1)));
    GP_CUDA(c, cudaMemcpyAsync(c->sched.p, d_sched, 24 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(counts, so.counts, 12, cudaMemcpyDeviceToHost, st));
    return GP_OK;
}

// The two gp_build_*availability entries: the availability stage, then every non-NULL outs[k] gets row k % 3 of
// availableResources for k < 3 (first_fit: that of rescheduleExecutor's first-fit branch), of SchedulableResources for k >= 3.
static gp_status availability_out(gp_ctx* c, const gp_usage_input* in, bool first_fit, int64_t* const* outs, const char* who) {
    gp_status s = check_usage(c, in, who);
    if (s != GP_OK) return s;
    const int32_t n = in->n_nodes;
    if (n == 0) return GP_OK;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    long long *d_avail = nullptr, *d_sched = nullptr, *d_ff = nullptr;
    s = stage_availability(c, in, st, &d_avail, &d_sched, first_fit ? &d_ff : nullptr);
    if (s != GP_OK) return s;
    const size_t N = (size_t)n;
    const long long* src[2] = {first_fit ? d_ff : d_avail, d_sched};
    for (int k = 0; k < 6; ++k)
        if (outs[k]) GP_CUDA(c, cudaMemcpyAsync(outs[k], src[k / 3] + N * (size_t)(k % 3), 8 * N, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

extern "C" {

gp_status gp_potential_nodes(gp_ctx* c, const gp_sort_input* in, int32_t* driver_order, int32_t* n_driver,
                             int32_t* executor_order, int32_t* n_executor) {
    if (!c) return GP_ERR_INVALID;
    if (!in || in->n_nodes < 0 || in->n_zones < 1 || !n_driver || !n_executor ||
        (in->n_nodes > 0 && (!in->avail_cpu_milli || !in->avail_mem_bytes || !driver_order || !executor_order)))
        return fail(c, GP_ERR_INVALID, "gp_potential_nodes: missing arrays or bad sizes");
    const int32_t n = in->n_nodes;
    *n_driver = 0; *n_executor = 0;
    if (n == 0) return GP_OK;
    gp_status s = check_sort_ids(c, in, "gp_potential_nodes");
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    SortStage so{};
    s = stage_sort(c, in, nullptr, nullptr, nullptr, st, &so);
    if (s != GP_OK) return s;
    int32_t counts[3] = {0, 0, 0};
    GP_CUDA(c, cudaMemcpyAsync(counts, so.counts, 12, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(driver_order, so.drv, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(executor_order, so.exe, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    *n_driver = counts[0];
    *n_executor = counts[1];
    if (in->undefined_ties) *in->undefined_ties = counts[2];
    return GP_OK;
}

gp_status gp_build_availability(gp_ctx* c, const gp_usage_input* in, int64_t* avail_cpu, int64_t* avail_mem, int64_t* avail_gpu,
                                int64_t* sched_cpu, int64_t* sched_mem, int64_t* sched_gpu) {
    if (!c) return GP_ERR_INVALID;
    int64_t* const outs[6] = {avail_cpu, avail_mem, avail_gpu, sched_cpu, sched_mem, sched_gpu};
    return availability_out(c, in, false, outs, "gp_build_availability");
}

// availableResources of rescheduleExecutor's first-fit branch: the availability to upload before gp_reschedule_executors(min_frag = 0)
gp_status gp_build_reschedule_availability(gp_ctx* c, const gp_usage_input* in, int64_t* avail_cpu, int64_t* avail_mem, int64_t* avail_gpu) {
    if (!c) return GP_ERR_INVALID;
    int64_t* const outs[6] = {avail_cpu, avail_mem, avail_gpu, nullptr, nullptr, nullptr};
    return availability_out(c, in, true, outs, "gp_build_reschedule_availability");
}

// reservations -> availability -> priority orders -> slot layout, without leaving the device
gp_status gp_prepare_cluster(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, int32_t* n_driver, int32_t* n_executor) {
    if (!c) return GP_ERR_INVALID;
    if (n_driver) *n_driver = 0;
    if (n_executor) *n_executor = 0;
    long long *d_avail = nullptr, *d_sched = nullptr;
    SortStage so{};
    gp_status s = prepare_orders(c, usage, sort, "gp_prepare_cluster", &d_avail, &d_sched, &so);
    if (s != GP_OK) return s;
    cudaStream_t st = c->stream;
    GP_CUDA(c, c->exec_off.reserve(8)); GP_CUDA(c, c->drv_off.reserve(8));
    gp_offsets_from_counts<<<1, 32, 0, st>>>(so.counts, c->exec_off.as<int32_t>(), c->drv_off.as<int32_t>());
    gp_nodes dn{};
    dn.n_nodes = usage->n_nodes;
    dn.n_groups = 1;
    dn.exec_off = c->exec_off.as<int32_t>(); dn.exec_order = so.exe;
    dn.drv_off = c->drv_off.as<int32_t>(); dn.drv_order = so.drv;
    int32_t counts[3] = {0, 0, 0};
    s = prepare_snapshot(c, &dn, d_avail, d_sched, so, counts);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaStreamSynchronize(st));
    c->n_drv = counts[0]; c->n_exec = counts[1];
    c->have_eff_sched = true;           // SchedulableResources for gp_packing_efficiency (the zone entry points still want gp_set_schedulable)
    if (sort->undefined_ties) *sort->undefined_ties = counts[2];
    if (n_driver) *n_driver = counts[0];
    if (n_executor) *n_executor = counts[1];
    return GP_OK;
}

// reservations -> availability -> priority orders -> zone-grouped slot layout, without leaving the device
gp_status gp_prepare_cluster_zones(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, gp_zone_layout* layout) {
    if (!c) return GP_ERR_INVALID;
    if (!layout) return fail(c, GP_ERR_INVALID, "gp_prepare_cluster_zones: missing arrays or mismatched sizes");
    const int32_t kind = layout->kind;
    if (kind != GP_LAYOUT_SINGLE_AZ && kind != GP_LAYOUT_AZ_AWARE)
        return fail(c, GP_ERR_INVALID, "gp_prepare_cluster_zones: layout->kind must be GP_LAYOUT_SINGLE_AZ or GP_LAYOUT_AZ_AWARE");
    if (sort && sort->n_zones == 0x7fffffff) return fail(c, GP_ERR_INVALID, "gp_prepare_cluster_zones: n_zones too large");
    layout->n_zones = 0; layout->n_groups = 0; layout->n_driver = 0; layout->n_executor = 0;
    long long *d_avail = nullptr, *d_sched = nullptr;
    SortStage so{};
    gp_status s = prepare_orders(c, usage, sort, "gp_prepare_cluster_zones", &d_avail, &d_sched, &so);
    if (s != GP_OK) return s;
    cudaStream_t st = c->stream;
    c->zone_kind = -1;                                  // the held orders are overwritten below
    const int32_t n = usage->n_nodes;
    const size_t N = (size_t)n;
    // g_bound = sort->n_zones + 1 groups bound every layout; the slots are laid out for that many (the groups past the
    // last one are empty) so that the group count can stay on the device until the one synchronise below
    const size_t Zs = (size_t)sort->n_zones;
    const int32_t g_bound = sort->n_zones + 1;
    Arena ar{c->zoneprep};
    const size_t o_udrv = ar.take(4 * N), o_uexe = ar.take(4 * N), o_first = ar.take(4 * Zs), o_has = ar.take(Zs), o_zg = ar.take(4 * Zs),
                 o_zog = ar.take(4 * (Zs + 1)), o_rank = ar.take(4 * N), o_lk = ar.take(sizeof(LabelKey) * N), o_lks = ar.take(sizeof(LabelKey) * N),
                 o_pos = ar.take(4 * N), o_info = ar.take(4 * kZiWords);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    int32_t* udrv = (int32_t*)(b + o_udrv);
    int32_t* uexe = (int32_t*)(b + o_uexe);
    int32_t* info = (int32_t*)(b + o_info);
    int32_t* rank = (int32_t*)(b + o_rank);
    // the undivided orders outlive the sort's scratch, which the next gp_potential_nodes / gp_prepare_cluster reuses
    GP_CUDA(c, cudaMemcpyAsync(udrv, so.drv, 4 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(uexe, so.exe, 4 * N, cudaMemcpyDeviceToDevice, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_first, 0x7f, 4 * Zs, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_has, 0, Zs, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_zg, 0xff, 4 * Zs, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_zog, 0xff, 4 * (Zs + 1), st));
    GP_CUDA(c, cudaMemsetAsync(info, 0, 4 * kZiWords, st));
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int32_t az = kind == GP_LAYOUT_AZ_AWARE ? 1 : 0;
    gp_zone_mark<<<nb, T, 0, st>>>(n, so.counts, udrv, uexe, so.zone, (int32_t*)(b + o_first), (uint8_t*)(b + o_has));
    gp_zone_candidates<<<1, 1024, 0, st>>>(so.counts, udrv, so.zone, (const int32_t*)(b + o_first), (const uint8_t*)(b + o_has),
                                           (int32_t*)(b + o_zg), (int32_t*)(b + o_zog), info);
    gp_group_rank<<<nb, T, 0, st>>>(n, so.counts, udrv, uexe, so.zone, (const int32_t*)(b + o_zg), az, info, rank);
    GP_CUDA(c, cudaGetLastError());
    // the grouped orders and their offsets
    GP_CUDA(c, c->exec_order.reserve(4 * (N + 1))); GP_CUDA(c, c->drv_order.reserve(4 * (N + 1)));
    GP_CUDA(c, c->exec_off.reserve(4 * ((size_t)g_bound + 1))); GP_CUDA(c, c->drv_off.reserve(4 * ((size_t)g_bound + 1)));
    LabelKey* lk = (LabelKey*)(b + o_lk);
    LabelKey* lks = (LabelKey*)(b + o_lks);
    int32_t* pos = (int32_t*)(b + o_pos);
    launch_label_resort(n, so.counts, udrv, rank, lk, lks, pos, c->drv_order.as<int32_t>(), st);
    launch_label_resort(n, so.counts + 1, uexe, rank, lk, lks, pos, c->exec_order.as<int32_t>(), st);
    gp_group_offsets<<<(unsigned)((g_bound + T) / T), T, 0, st>>>(g_bound, so.counts, c->drv_order.as<int32_t>(), c->exec_order.as<int32_t>(),
                                                                  rank, az, c->exec_off.as<int32_t>(), c->drv_off.as<int32_t>(), info);
    GP_CUDA(c, cudaGetLastError());
    gp_nodes dn{};
    dn.n_nodes = n;
    dn.n_groups = g_bound;
    dn.exec_off = c->exec_off.as<int32_t>(); dn.exec_order = c->exec_order.as<int32_t>();
    dn.drv_off = c->drv_off.as<int32_t>(); dn.drv_order = c->drv_order.as<int32_t>();
    int32_t counts[3] = {0, 0, 0}, hinfo[kZiWords] = {};
    s = prepare_snapshot(c, &dn, d_avail, d_sched, so, counts);
    if (s != GP_OK) return s;
    GP_CUDA(c, cudaMemcpyAsync(hinfo, info, sizeof(hinfo), cudaMemcpyDeviceToHost, st));
    if (layout->zone_of_group) GP_CUDA(c, cudaMemcpyAsync(layout->zone_of_group, b + o_zog, 4 * (Zs + 1), cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    c->n_groups = hinfo[kZiGroups]; c->n_exec = hinfo[kZiExec]; c->n_drv = hinfo[kZiDrv];
    c->have_sched = true;
    c->have_eff_sched = true;
    c->zone_orders = gp_az_orders{hinfo[kZiZones], counts[1], uexe, counts[0], udrv};
    c->zone_kind = kind;
    if (sort->undefined_ties) *sort->undefined_ties = counts[2];
    layout->n_zones = hinfo[kZiZones]; layout->n_groups = hinfo[kZiGroups];
    layout->n_driver = counts[0]; layout->n_executor = counts[1];
    // the grouped layout itself only when asked: its sizes are known now
    const size_t ob = 4 * (size_t)(hinfo[kZiGroups] + 1);
    if (layout->exec_off) GP_CUDA(c, cudaMemcpyAsync(layout->exec_off, c->exec_off.p, ob, cudaMemcpyDeviceToHost, st));
    if (layout->drv_off) GP_CUDA(c, cudaMemcpyAsync(layout->drv_off, c->drv_off.p, ob, cudaMemcpyDeviceToHost, st));
    if (layout->exec_order && c->n_exec) GP_CUDA(c, cudaMemcpyAsync(layout->exec_order, c->exec_order.p, 4 * (size_t)c->n_exec, cudaMemcpyDeviceToHost, st));
    if (layout->drv_order && c->n_drv) GP_CUDA(c, cudaMemcpyAsync(layout->drv_order, c->drv_order.p, 4 * (size_t)c->n_drv, cudaMemcpyDeviceToHost, st));
    if (layout->exec_off || layout->drv_off || layout->exec_order || layout->drv_order) GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

// rescheduleExecutor's node choice for a batch of executors (SURVEY 8f row f4); see gangpack_resched.cuh
gp_status gp_reschedule_executors(gp_ctx* c, const gp_reschedule* in, int32_t* node_out) {
    if (!c) return GP_ERR_INVALID;
    if (!c->have_snapshot) return fail(c, GP_ERR_NO_SNAPSHOT, "gp_reschedule_executors: gp_set_snapshot first");
    if (!in || in->n_execs < 0 || (in->n_execs > 0 && (!in->exe_cpu_milli || !in->exe_mem_bytes || !node_out)))
        return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: missing arrays or bad sizes");
    const int32_t q = in->n_execs;
    if (q == 0) return GP_OK;
    const bool mf = in->min_frag != 0;
    const bool has_res = mf && in->reserved_cpu_milli;
    const bool has_host = mf && in->host_off;
    if (has_res && !in->reserved_mem_bytes) return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: reserved_mem_bytes missing");
    // host validation (O(q + n_nodes + hosted)): the exact-int64 domain, non-negative requests, CSR shape
    gp_status chk = check_requests(c, q, in->exe_cpu_milli, in->exe_mem_bytes, in->exe_gpu, "gp_reschedule_executors");
    if (chk != GP_OK) return chk;
    for (int32_t i = 0; i < q; ++i)
        if (in->group && (in->group[i] < 0 || in->group[i] >= c->n_groups)) return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: instance group out of range");
    if (has_res)
        for (int32_t n = 0; n < c->n_nodes; ++n) {
            const int64_t v[3] = {in->reserved_cpu_milli[n], in->reserved_mem_bytes[n], in->reserved_gpu ? in->reserved_gpu[n] : 0};
            for (int64_t x : v)
                if (x >= kMaxQuantity || x <= -kMaxQuantity) return fail(c, GP_ERR_UNREPRESENTABLE, "gp_reschedule_executors: |reserved| >= 2^61");
        }
    int64_t hosted = 0;
    if (has_host && (chk = check_hosting(c, in, c->n_nodes, &hosted, "gp_reschedule_executors")) != GP_OK) return chk;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t Q = (size_t)q, N = (size_t)c->n_nodes, H = (size_t)hosted;
    Arena ar{c->reschedbuf};
    const size_t o_exe = ar.take(8 * 3 * Q), o_res = ar.take(8 * 3 * N), o_hoff = ar.take(8 * (Q + 1)), o_grp = ar.take(4 * Q),
                 o_hn = ar.take(4 * (H + 1)), o_out = ar.take(4 * Q), o_err = ar.take(8);
    GP_CUDA(c, ar.reserve());
    char* base = ar.base();
    int64_t* d_exe = reinterpret_cast<int64_t*>(base + o_exe);
    int64_t* d_res = reinterpret_cast<int64_t*>(base + o_res);
    int64_t* d_hoff = reinterpret_cast<int64_t*>(base + o_hoff);
    int32_t* d_grp = reinterpret_cast<int32_t*>(base + o_grp);
    int32_t* d_hn = reinterpret_cast<int32_t*>(base + o_hn);
    int32_t* d_out = reinterpret_cast<int32_t*>(base + o_out);
    int* d_err = reinterpret_cast<int*>(base + o_err);
    GP_CUDA(c, cudaMemsetAsync(d_err, 0, 8, st));
    GP_CUDA(c, cudaMemcpyAsync(d_exe, in->exe_cpu_milli, 8 * Q, cudaMemcpyHostToDevice, st));
    GP_CUDA(c, cudaMemcpyAsync(d_exe + Q, in->exe_mem_bytes, 8 * Q, cudaMemcpyHostToDevice, st));
    if (in->exe_gpu) GP_CUDA(c, cudaMemcpyAsync(d_exe + 2 * Q, in->exe_gpu, 8 * Q, cudaMemcpyHostToDevice, st));
    if (in->group) GP_CUDA(c, cudaMemcpyAsync(d_grp, in->group, 4 * Q, cudaMemcpyHostToDevice, st));
    if (has_res && N) {
        GP_CUDA(c, cudaMemcpyAsync(d_res, in->reserved_cpu_milli, 8 * N, cudaMemcpyHostToDevice, st));
        GP_CUDA(c, cudaMemcpyAsync(d_res + N, in->reserved_mem_bytes, 8 * N, cudaMemcpyHostToDevice, st));
        if (in->reserved_gpu) GP_CUDA(c, cudaMemcpyAsync(d_res + 2 * N, in->reserved_gpu, 8 * N, cudaMemcpyHostToDevice, st));
    }
    if (has_host) {
        GP_CUDA(c, cudaMemcpyAsync(d_hoff, in->host_off, 8 * (Q + 1), cudaMemcpyHostToDevice, st));
        if (H) GP_CUDA(c, cudaMemcpyAsync(d_hn, in->host_nodes, 4 * H, cudaMemcpyHostToDevice, st));
    }
    ReschedIn ri{};
    ri.exe_cpu = d_exe; ri.exe_mem = d_exe + Q; ri.exe_gpu = in->exe_gpu ? d_exe + 2 * Q : nullptr;
    ri.group = in->group ? d_grp : nullptr;
    ri.res_cpu = has_res ? d_res : nullptr; ri.res_mem = has_res ? d_res + N : nullptr;
    ri.res_gpu = (has_res && in->reserved_gpu) ? d_res + 2 * N : nullptr;
    ri.host_off = has_host ? d_hoff : nullptr; ri.host_nodes = d_hn;
    ri.node_slot = c->node_slot.as<int32_t>();
    ri.n_execs = q;
    const Snapshot s = make_snapshot(c);
    const int T = 256;
    int64_t blocks = ((int64_t)q * 32 + T - 1) / T;
    const int64_t max_blocks = (int64_t)c->sm_count * 8;
    if (blocks > max_blocks) blocks = max_blocks;
    if (mf) gp_reschedule_kernel<true><<<(int)blocks, T, 0, st>>>(s, ri, d_out, d_err);
    else gp_reschedule_kernel<false><<<(int)blocks, T, 0, st>>>(s, ri, d_out, d_err);
    GP_CUDA(c, cudaGetLastError());
    int err = 0;
    GP_CUDA(c, cudaMemcpyAsync(node_out, d_out, 4 * Q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (err) return fail(c, GP_ERR_INVALID, "gp_reschedule_executors: instance group out of range");
    return GP_OK;
}

// rescheduleExecutor from the reservations to the node choice (SURVEY 8f row f4); see gangpack_reschedprep.cuh
gp_status gp_reschedule_from_reservations(gp_ctx* c, const gp_usage_input* usage, const gp_sort_input* sort, const gp_reschedule_scope* scope,
                                          const gp_reschedule* in, int32_t* node_out, uint8_t* ambiguous) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_reschedule_from_reservations";
    auto bad = [&](gp_status st, const char* what) { return fail(c, st, std::string(who) + ": " + what); };
    gp_status s = check_usage(c, usage, who);
    if (s != GP_OK) return s;
    if (!sort || !in || usage->n_nodes != sort->n_nodes || sort->n_zones < 1 ||
        in->n_execs < 0 || (in->n_execs > 0 && (!in->exe_cpu_milli || !in->exe_mem_bytes || !node_out)))
        return bad(GP_ERR_INVALID, "missing arrays or mismatched sizes");
    const int32_t n = usage->n_nodes, q = in->n_execs;
    if (n == 0) return bad(GP_ERR_INVALID, "empty node table");
    if (in->reserved_cpu_milli || in->reserved_mem_bytes || in->reserved_gpu)
        return bad(GP_ERR_INVALID, "reserved_* must be NULL (the overhead of the node table is the reserved amount)");
    const int32_t keep = scope ? scope->keep_topology_zone : -1;
    if (keep < -1) return bad(GP_ERR_INVALID, "scope->keep_topology_zone must be -1 or a zone id");
    if (keep >= 0) {
        if (!scope->topology_zone) return bad(GP_ERR_INVALID, "scope->topology_zone missing");
        for (int32_t i = 0; i < n; ++i)
            if (scope->topology_zone[i] < 0)
                return bad(GP_ERR_INVALID, "filterNodesToZone: a node has no topology.kubernetes.io/zone label (topology_zone == -1), "
                                           "unable to make scheduling decisions based on AZ");
    }
    if ((s = check_sort_ids(c, sort, who)) != GP_OK) return s;
    const bool mf = in->min_frag != 0;
    const bool has_host = mf && in->host_off;
    if ((s = check_requests(c, q, in->exe_cpu_milli, in->exe_mem_bytes, in->exe_gpu, who)) != GP_OK) return s;
    for (int32_t i = 0; i < q; ++i)
        if (in->group && in->group[i] != 0) return bad(GP_ERR_INVALID, "instance group out of range (one node table: group must be 0)");
    int64_t hosted = 0;
    if (has_host && (s = check_hosting(c, in, n, &hosted, who)) != GP_OK) return s;
    if (q == 0) return GP_OK;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    // availability: one scatter of the reservations, one pass per node (usagebuf is scratch of the f2 stage only)
    long long *d_avail = nullptr, *d_sched = nullptr, *d_ff = nullptr;
    const long long* d_over[3] = {nullptr, nullptr, nullptr};
    s = stage_availability(c, usage, st, &d_avail, &d_sched, mf ? nullptr : &d_ff, d_over);
    if (s != GP_OK) return s;
    const size_t N = (size_t)n, Q = (size_t)q, H = (size_t)hosted, Z = (size_t)sort->n_zones;
    const bool zoned = sort->zone_id != nullptr && sort->n_zones > 1;
    Arena ar{c->reschedprep};
    const size_t o_tot = ar.take(16 * Z), o_prio = ar.take(4 * Z), o_zone = ar.take(4 * N), o_nr = ar.take(4 * N), o_fu = ar.take(N),
                 o_fr = ar.take(N), o_lr = ar.take(4 * N), o_tz = ar.take(4 * N), o_rec = ar.take(sizeof(RpNode) * N), o_exe = ar.take(24 * Q),
                 o_hoff = ar.take(8 * (Q + 1)), o_hn = ar.take(4 * (H + 1)), o_out = ar.take(4 * Q), o_amb = ar.take(Q);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    if (zoned) GP_CUDA(c, ar.upload(o_zone, sort->zone_id, 4 * N, st));
    if (sort->name_rank) GP_CUDA(c, ar.upload(o_nr, sort->name_rank, 4 * N, st));
    if (sort->unschedulable) GP_CUDA(c, ar.upload(o_fu, sort->unschedulable, N, st));
    if (sort->ready) GP_CUDA(c, ar.upload(o_fr, sort->ready, N, st));
    if (sort->executor_label_rank) GP_CUDA(c, ar.upload(o_lr, sort->executor_label_rank, 4 * N, st));
    if (keep >= 0) GP_CUDA(c, ar.upload(o_tz, scope->topology_zone, 4 * N, st));
    GP_CUDA(c, ar.upload(o_exe, in->exe_cpu_milli, 8 * Q, st));
    GP_CUDA(c, ar.upload(o_exe + 8 * Q, in->exe_mem_bytes, 8 * Q, st));
    if (in->exe_gpu) GP_CUDA(c, ar.upload(o_exe + 16 * Q, in->exe_gpu, 8 * Q, st));
    else GP_CUDA(c, cudaMemsetAsync(b + o_exe + 16 * Q, 0, 8 * Q, st));
    if (has_host) {
        GP_CUDA(c, ar.upload(o_hoff, in->host_off, 8 * (Q + 1), st));
        if (H) GP_CUDA(c, ar.upload(o_hn, in->host_nodes, 4 * H, st));
    }
    const int T = 256;
    const int nb = (n + T - 1) / T;
    const int32_t* tz = keep >= 0 ? (const int32_t*)(b + o_tz) : nullptr;
    if (zoned) {
        GP_CUDA(c, cudaMemsetAsync(b + o_tot, 0, 16 * Z, st));
        gp_rp_zone_totals<<<nb, T, 0, st>>>(n, d_avail, d_avail + N, (const int32_t*)(b + o_zone), keep, tz, (unsigned long long*)(b + o_tot));
        gp_zone_priority<<<(sort->n_zones + T - 1) / T, T, 0, st>>>(sort->n_zones, (const unsigned long long*)(b + o_tot), (int32_t*)(b + o_prio));
    }
    RpNodeIn ni{};
    ni.avail = d_avail; ni.ff = d_ff;
    for (int d = 0; d < 3; ++d) ni.over[d] = d_over[d];
    ni.zone = zoned ? (const int32_t*)(b + o_zone) : nullptr;
    ni.prio = (const int32_t*)(b + o_prio);
    ni.name_rank = sort->name_rank ? (const int32_t*)(b + o_nr) : nullptr;
    ni.unschedulable = sort->unschedulable ? (const uint8_t*)(b + o_fu) : nullptr;
    ni.ready = sort->ready ? (const uint8_t*)(b + o_fr) : nullptr;
    ni.label_rank = sort->executor_label_rank ? (const int32_t*)(b + o_lr) : nullptr;
    ni.tz = tz; ni.keep = keep; ni.n = n;
    RpNode* rec = (RpNode*)(b + o_rec);
    gp_rp_nodes<<<nb, T, 0, st>>>(ni, rec);
    RpDecideIn di{};
    di.exe = (const int64_t*)(b + o_exe);
    di.host_off = has_host ? (const int64_t*)(b + o_hoff) : nullptr;
    di.host_nodes = (const int32_t*)(b + o_hn);
    di.n = n; di.q = q;
    // one CTA per executor; the grid is capped at 8 CTAs per SM's worth of executors and grid-strides over the rest.  The cap
    // only sizes the grid: registers bound residency (gp_rp_decide<true>: 78 x 256 threads -> 3 CTAs per SM; <false>: 48 -> 5),
    // so the CTAs beyond that wait for a free slot
    const int blocks = (int)std::min<int64_t>(q, (int64_t)c->sm_count * 8);
    int32_t* d_out = (int32_t*)(b + o_out);
    uint8_t* d_amb = ambiguous ? (uint8_t*)(b + o_amb) : nullptr;
    if (mf) gp_rp_decide<true><<<blocks, kRpThreads, 0, st>>>(rec, di, d_out, d_amb);
    else gp_rp_decide<false><<<blocks, kRpThreads, 0, st>>>(rec, di, d_out, d_amb);
    GP_CUDA(c, cudaGetLastError());
    GP_CUDA(c, cudaMemcpyAsync(node_out, d_out, 4 * Q, cudaMemcpyDeviceToHost, st));
    if (ambiguous) GP_CUDA(c, cudaMemcpyAsync(ambiguous, d_amb, Q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return GP_OK;
}

}  // extern "C"

// ---- required node affinity and the marker's capacity checks (gangpack_affinity.cuh, gangpack_capacity.cuh) ---------------
// Host checks of the label offsets and of the affinity programs (small); each label entry is checked by gp_aff_match itself.
static gp_status check_affinity(gp_ctx* c, const gp_node_labels* L, const gp_node_affinities* P, const char* who) {
    auto bad = [&](const char* what) { return fail(c, GP_ERR_INVALID, std::string(who) + ": " + what); };
    if (!L || !P || L->n_nodes < 0 || L->n_keys < 0 || L->n_values < 0 || P->n_aff < 0 || !L->label_off || !P->sel_off ||
        !P->term_off || !P->term_req_off || !P->req_val_off || (P->n_aff > 0 && !P->has_required) || (L->label_int_ok && !L->label_int))
        return bad("missing arrays or negative sizes");
    auto csr = [](const int64_t* off, int64_t n) {      // off[0] = 0, non-decreasing
        if (off[0] != 0) return false;
        for (int64_t i = 0; i < n; ++i) if (off[i + 1] < off[i]) return false;
        return true;
    };
    const int32_t n = L->n_nodes, A = P->n_aff;
    if (!csr(L->label_off, n)) return bad("label_off does not start at 0 or decreases");
    if (L->label_off[n] > 0 && (!L->label_key || !L->label_val)) return bad("missing arrays or negative sizes");
    if (!csr(P->sel_off, A) || !csr(P->term_off, A)) return bad("sel_off or term_off does not start at 0 or decreases");
    const int64_t ns = P->sel_off[A], nt = P->term_off[A];
    if (!csr(P->term_req_off, nt)) return bad("term_req_off does not start at 0 or decreases");
    const int64_t nr = P->term_req_off[nt];
    if (!csr(P->req_val_off, nr)) return bad("req_val_off does not start at 0 or decreases");
    const int64_t nv = P->req_val_off[nr];
    if ((ns > 0 && (!P->sel_key || !P->sel_val)) || (nr > 0 && (!P->req_op || !P->req_key || !P->req_int)) || (nv > 0 && !P->req_val))
        return bad("missing arrays or negative sizes");
    for (int64_t t = 0; t < ns; ++t)
        if (P->sel_key[t] < 0 || P->sel_key[t] >= L->n_keys || P->sel_val[t] < 0 || P->sel_val[t] >= L->n_values)
            return bad("node selector key or value id out of range");
    for (int64_t r = 0; r < nr; ++r) {
        const int32_t op = P->req_op[r];
        if (op < GP_AFF_IN || op > GP_AFF_FIELD_NAME_NOT_IN) return bad("requirement operator out of range");
        if (op >= GP_AFF_FIELD_NAME_IN) {
            if (P->req_int[r] < -1 || P->req_int[r] >= n) return bad("metadata.name node index out of range (-1 or 0..n_nodes-1)");
            continue;
        }
        if (P->req_key[r] < 0 || P->req_key[r] >= L->n_keys) return bad("requirement key id out of range");
        for (int64_t v = P->req_val_off[r]; v < P->req_val_off[r + 1]; ++v) {
            if (P->req_val[v] < 0 || P->req_val[v] >= L->n_values) return bad("requirement value id out of range");
            if (v > P->req_val_off[r] && P->req_val[v] <= P->req_val[v - 1]) return bad("requirement values not strictly ascending");
        }
    }
    return GP_OK;
}

// Device staging of the labels and programs, and the match launches
struct AffStage {
    size_t o_loff, o_lkey, o_lval, o_lok, o_lint, o_soff, o_skey, o_sval, o_hreq, o_toff, o_troff, o_terr, o_rop, o_rkey, o_rint,
        o_rvoff, o_rval, o_nm, o_ne, o_err;
    int64_t nl, ns, nt, nr, nv;
    int32_t n, A, words;
    AffLabelsIn L{};
    AffProgIn P{};

    void take(Arena& ar, const gp_node_labels* l, const gp_node_affinities* p) {
        n = l->n_nodes; A = p->n_aff; words = (n + 31) / 32;
        nl = l->label_off[n]; ns = p->sel_off[A]; nt = p->term_off[A]; nr = p->term_req_off[nt]; nv = p->req_val_off[nr];
        const size_t N1 = (size_t)n + 1, A1 = (size_t)A + 1;
        o_loff = ar.take(8 * N1); o_lkey = ar.take(4 * nl); o_lval = ar.take(4 * nl); o_lok = ar.take(nl); o_lint = ar.take(8 * nl);
        o_soff = ar.take(8 * A1); o_skey = ar.take(4 * ns); o_sval = ar.take(4 * ns); o_hreq = ar.take(A);
        o_toff = ar.take(8 * A1); o_troff = ar.take(8 * (nt + 1)); o_terr = ar.take(nt);
        o_rop = ar.take(4 * nr); o_rkey = ar.take(4 * nr); o_rint = ar.take(8 * nr); o_rvoff = ar.take(8 * (nr + 1)); o_rval = ar.take(4 * nv);
        o_nm = ar.take(4 * (size_t)A); o_ne = ar.take(4 * (size_t)A); o_err = ar.take(8);
    }
    // uploads, zeroes the counters and the error word
    cudaError_t upload(const Arena& ar, const gp_node_labels* l, const gp_node_affinities* p, cudaStream_t st) {
        char* b = ar.base();
        struct Piece { size_t o; const void* src; size_t bytes; };
        const Piece pieces[] = {
            {o_loff, l->label_off, 8 * ((size_t)n + 1)}, {o_lkey, l->label_key, 4 * (size_t)nl}, {o_lval, l->label_val, 4 * (size_t)nl},
            {o_lok, l->label_int_ok, (size_t)nl}, {o_lint, l->label_int, 8 * (size_t)nl},
            {o_soff, p->sel_off, 8 * ((size_t)A + 1)}, {o_skey, p->sel_key, 4 * (size_t)ns}, {o_sval, p->sel_val, 4 * (size_t)ns},
            {o_hreq, p->has_required, (size_t)A}, {o_toff, p->term_off, 8 * ((size_t)A + 1)},
            {o_troff, p->term_req_off, 8 * ((size_t)nt + 1)}, {o_terr, p->term_parse_error, (size_t)nt},
            {o_rop, p->req_op, 4 * (size_t)nr}, {o_rkey, p->req_key, 4 * (size_t)nr}, {o_rint, p->req_int, 8 * (size_t)nr},
            {o_rvoff, p->req_val_off, 8 * ((size_t)nr + 1)}, {o_rval, p->req_val, 4 * (size_t)nv}};
        for (const Piece& pc : pieces) {
            if (pc.bytes == 0) continue;
            const cudaError_t e = pc.src ? ar.upload(pc.o, pc.src, pc.bytes, st) : cudaMemsetAsync(b + pc.o, 0, pc.bytes, st);
            if (e != cudaSuccess) return e;
        }
        L.n = n; L.n_keys = l->n_keys; L.n_values = l->n_values;
        L.off = (const long long*)(b + o_loff); L.key = (const int32_t*)(b + o_lkey); L.val = (const int32_t*)(b + o_lval);
        L.int_ok = l->label_int_ok ? (const uint8_t*)(b + o_lok) : nullptr; L.ival = (const long long*)(b + o_lint);
        P.n_aff = A;
        P.sel_off = (const long long*)(b + o_soff); P.sel_key = (const int32_t*)(b + o_skey); P.sel_val = (const int32_t*)(b + o_sval);
        P.has_required = (const uint8_t*)(b + o_hreq); P.term_off = (const long long*)(b + o_toff);
        P.term_req_off = (const long long*)(b + o_troff); P.term_err = (const uint8_t*)(b + o_terr);
        P.req_op = (const int32_t*)(b + o_rop); P.req_key = (const int32_t*)(b + o_rkey); P.req_int = (const long long*)(b + o_rint);
        P.req_val_off = (const long long*)(b + o_rvoff); P.req_val = (const int32_t*)(b + o_rval);
        // n_match, n_error and the error word; the labels are checked once here, whatever the number of affinities
        cudaError_t e = cudaMemsetAsync(b + o_nm, 0, 4 * (size_t)A, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(b + o_ne, 0, 4 * (size_t)A, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(b + o_err, 0, 8, st);
        if (e == cudaSuccess && n > 0) gp_aff_labels<<<(unsigned)((n + kAffThreads - 1) / kAffThreads), kAffThreads, 0, st>>>(L, (int*)(b + o_err));
        return e;
    }
    // affinities [a0, a0 + k) into member rows 0..k-1
    void match(const Arena& ar, uint32_t* member, int32_t a0, int32_t k, cudaStream_t st) const {
        if (n == 0) return;
        char* b = ar.base();
        AffOut out{member, (int32_t*)(b + o_nm), (int32_t*)(b + o_ne), words, a0};
        for (int32_t y = 0; y < k; y += 65535) {
            const dim3 grid((unsigned)((n + kAffThreads - 1) / kAffThreads), (unsigned)std::min(k - y, 65535));
            gp_aff_match<<<grid, kAffThreads, 0, st>>>(L, P, out, a0 + y);
        }
    }
    gp_status label_error(gp_ctx* c, int herr, const char* who) const {
        if (herr & kAffErrLabelKey) return fail(c, GP_ERR_INVALID, std::string(who) + ": label key id out of range or the keys of a node not strictly ascending");
        if (herr & kAffErrLabelVal) return fail(c, GP_ERR_INVALID, std::string(who) + ": label value id out of range");
        return GP_OK;
    }
};

// DoesPodExceedClusterCapacity for a batch of stale drivers, any packer; the node sets are the node_group classes (aff ==
// NULL) or the affinities' matches
static gp_status capacity_run(gp_ctx* c, const char* who, const gp_capacity_nodes* nodes, const gp_node_labels* labels,
                              const gp_node_affinities* aff, const gp_apps* a, gp_binpacker packer, uint8_t* exceeds,
                              uint8_t* affinity_error) {
    auto bad = [&](gp_status st, const char* what) { return fail(c, st, std::string(who) + ": " + what); };
    if (!aff) {
        if (!nodes || !a || nodes->n_nodes < 0 || a->n_apps < 0 || nodes->n_groups < 1 || (nodes->zone_id && nodes->n_zones < 1) ||
            (nodes->n_nodes > 0 && (!nodes->alloc_cpu_milli || !nodes->alloc_mem_bytes)) ||
            (a->n_apps > 0 && (!a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !exceeds)))
            return bad(GP_ERR_INVALID, "missing arrays or bad sizes (n_groups >= 1; n_zones >= 1 with zone_id)");
    } else {
        if (!nodes || !a || nodes->n_nodes < 0 || a->n_apps < 0 || (nodes->zone_id && nodes->n_zones < 1) ||
            (nodes->n_nodes > 0 && (!nodes->alloc_cpu_milli || !nodes->alloc_mem_bytes)) ||
            (a->n_apps > 0 && (!a->drv_cpu_milli || !a->drv_mem_bytes || !a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count ||
                               !a->group || !exceeds)))
            return bad(GP_ERR_INVALID, "missing arrays or bad sizes (group required; n_zones >= 1 with zone_id)");
        if (nodes->node_group) return bad(GP_ERR_INVALID, "node_group must be NULL: the node sets are the affinities' matches");
        if (!labels || labels->n_nodes != nodes->n_nodes) return bad(GP_ERR_INVALID, "labels->n_nodes != nodes->n_nodes");
        const gp_status s = check_affinity(c, labels, aff, who);
        if (s != GP_OK) return s;
    }
    if ((int)packer < GP_BP_TIGHTLY_PACK || (int)packer > GP_BP_SINGLE_AZ_MINIMAL_FRAGMENTATION) return bad(GP_ERR_INVALID, "unknown packer");
    const int32_t n = nodes->n_nodes, Q = a->n_apps;
    const int32_t Z = nodes->zone_id ? nodes->n_zones : 1, G = aff ? aff->n_aff : nodes->n_groups;
    if (!aff && (int64_t)(G + 1) * Z > (int64_t)INT32_MAX / 2) return bad(GP_ERR_INVALID, "(n_groups + 1) * n_zones too large");
    if (aff && (int64_t)Z > (int64_t)INT32_MAX / 2) return bad(GP_ERR_INVALID, "n_zones too large");
    // classes per chunk: node_group -> its own class and the all-nodes class; affinities -> as many as keep K n and K Z
    // within kCapEntries (at least one)
    const int32_t K = !aff ? 2 : (int32_t)std::max<int64_t>(1, std::min<int64_t>(std::max(G, 1), kCapEntries / std::max<int64_t>({(int64_t)n, (int64_t)Z, 1})));
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t N = (size_t)n, q = (size_t)Q, E = (size_t)K * N, B = aff ? (size_t)K * (size_t)Z : (size_t)(G + 1) * (size_t)Z;
    size_t H = 64;
    while (H < 2 * q) H <<= 1;                          // more slots than drivers: every probe ends
    const size_t n_segs = E / kCapSeg + B + 1;
    // buckets of more than kCapSeg nodes in a chunk: at most E / (kCapSeg + 1), whatever the number of zones
    const int32_t ms_stride = (int32_t)std::max<size_t>(1, E / ((size_t)kCapSeg + 1));
    const int32_t pairs_per_chunk = (int32_t)std::max<int64_t>(1, std::min<int64_t>(std::max(Q, 1), kCapSlotEntries / ms_stride));
    const size_t A = (size_t)pairs_per_chunk * (size_t)ms_stride;
    const size_t q1 = std::max<size_t>(q, 1);
    Arena ar{c->capprep};
    const size_t o_alloc = ar.take(24 * N), o_over = ar.take(24 * N), o_zone = ar.take(4 * N), o_grp = ar.take(4 * N), o_key = ar.take(4 * E),
                 o_rank = ar.take(4 * E), o_zst = ar.take(4 * N), o_staged = ar.take(24 * N), o_sched = ar.take(24 * E), o_bcnt = ar.take(4 * B),
                 o_boff = ar.take(4 * (B + 1)), o_soff = ar.take(4 * (B + 1)), o_moff = ar.take(4 * (B + 1)), o_segs = ar.take(sizeof(CapSeg) * n_segs),
                 o_q = ar.take(48 * q), o_cnt = ar.take(4 * q), o_ag = ar.take(4 * q), o_hash = ar.take(sizeof(CapEntry) * H),
                 o_pairs = ar.take(sizeof(CapPair) * q), o_np = ar.take(8), o_err = ar.take(8), o_ap = ar.take(4 * q),
                 o_pref = ar.take(8 * (q + 1)), o_slots = ar.take(sizeof(CapSlot) * A), o_T = ar.take(8 * q1),
                 o_M = ar.take(8 * q1), o_zb = ar.take(8 * q1), o_out = ar.take(q1);
    AffStage as{};
    size_t o_member = 0;
    if (aff) { as.take(ar, labels, aff); o_member = ar.take(4 * (size_t)K * (size_t)as.words); }
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    // n_pairs and the error word are adjacent: one memset clears both
    GP_CUDA(c, cudaMemsetAsync(b + o_hash, 0, sizeof(CapEntry) * H, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_np, 0, o_ap - o_np, st));
    if (aff) GP_CUDA(c, as.upload(ar, labels, aff, st));
    CapScratch s{};
    s.key = (int32_t*)(b + o_key); s.rank = (int32_t*)(b + o_rank); s.zone = (int32_t*)(b + o_zst); s.bucket_cnt = (int32_t*)(b + o_bcnt);
    s.bucket_off = (int32_t*)(b + o_boff); s.seg_off = (int32_t*)(b + o_soff); s.ms_off = (int32_t*)(b + o_moff);
    for (int d = 0; d < 3; ++d) { s.staged[d] = (long long*)(b + o_staged) + d * N; s.sched[d] = (long long*)(b + o_sched) + d * E; }
    s.segs = (CapSeg*)(b + o_segs); s.err = (int*)(b + o_err);
    s.Z = Z; s.G = G; s.n = n;
    const int T = 256;
    CapClassesIn ci{};
    if (n > 0) {
        CapNodesIn ni{};
        ni.n = n;
        const int64_t* cols[6] = {nodes->alloc_cpu_milli, nodes->alloc_mem_bytes, nodes->alloc_gpu,
                                  nodes->overhead_cpu_milli, nodes->overhead_mem_bytes, nodes->overhead_gpu};
        for (int d = 0; d < 6; ++d) {
            if (!cols[d]) continue;
            const size_t o = (d < 3 ? o_alloc : o_over) + 8 * N * (size_t)(d % 3);
            GP_CUDA(c, ar.upload(o, cols[d], 8 * N, st));
            (d < 3 ? ni.alloc : ni.over)[d % 3] = (const long long*)(b + o);
        }
        if (nodes->zone_id) { GP_CUDA(c, ar.upload(o_zone, nodes->zone_id, 4 * N, st)); ni.zone = (const int32_t*)(b + o_zone); }
        if (nodes->node_group) { GP_CUDA(c, ar.upload(o_grp, nodes->node_group, 4 * N, st)); ni.group = (const int32_t*)(b + o_grp); }
        ci.group = ni.group;
        gp_cc_nodes<<<(unsigned)((N + T - 1) / T), T, 0, st>>>(ni, s);
    }
    CapAppsIn ai{};
    ai.n = Q;
    const int64_t* qcols[6] = {a->drv_cpu_milli, a->drv_mem_bytes, a->drv_gpu, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu};
    for (int t = 0; t < 6; ++t) {
        if (!qcols[t]) continue;
        GP_CUDA(c, ar.upload(o_q + 8 * q * (size_t)t, qcols[t], 8 * q, st));
        ai.q[t] = (const long long*)(b + o_q) + q * (size_t)t;
    }
    if (Q > 0) GP_CUDA(c, ar.upload(o_cnt, a->exe_count, 4 * q, st));
    ai.count = (const int32_t*)(b + o_cnt);
    if (a->group && Q > 0) { GP_CUDA(c, ar.upload(o_ag, a->group, 4 * q, st)); ai.group = (const int32_t*)(b + o_ag); }
    ai.n_groups = G;
    ai.min_group = aff ? 0 : -1;
    ai.hash_mask = (uint32_t)(H - 1);
    CapPair* pairs = (CapPair*)(b + o_pairs);
    int32_t* n_pairs = (int32_t*)(b + o_np);
    int32_t* app_pair = (int32_t*)(b + o_ap);
    if (Q > 0) gp_cc_intern<<<(unsigned)((q + T - 1) / T), T, 0, st>>>(ai, (CapEntry*)(b + o_hash), pairs, n_pairs, app_pair, s.err);
    long long* pref = (long long*)(b + o_pref);
    CapPairOut po{(unsigned long long*)(b + o_T), (long long*)(b + o_M), (long long*)(b + o_zb)};
    CapPassIn pi{};
    pi.pairs = pairs; pi.n_pairs = n_pairs; pi.pref = pref; pi.out = po;
    pi.slots = (CapSlot*)(b + o_slots); pi.ms_stride = ms_stride;
    const int pass_blocks = c->sm_count * 8;
    if (aff) { ci.member = (const uint32_t*)(b + o_member); ci.words = as.words; }
    // node_group: one chunk of both entries of every node (a0 = -1); affinities: chunks of K classes, the last one possibly
    // shorter (none when there are no affinities: the nodes and drivers are still validated)
    const int32_t n_chunks = aff ? (G + K - 1) / K : 1;
    for (int32_t ch = 0; ch < n_chunks; ++ch) {
        const int32_t a0 = aff ? ch * K : -1, k = aff ? std::min(K, G - a0) : 2;
        s.a0 = a0; s.K = k; s.B = aff ? k * Z : (int32_t)B;
        if (aff) as.match(ar, (uint32_t*)(b + o_member), a0, k, st);
        GP_CUDA(c, cudaMemsetAsync(s.bucket_cnt, 0, 4 * (size_t)s.B, st));
        const size_t e = (size_t)k * N;
        if (n > 0) gp_cc_keys<<<(unsigned)((e + T - 1) / T), T, 0, st>>>(ci, s);
        gp_cc_bucket_scan<<<1, 1024, 0, st>>>(s);
        if (n > 0) gp_cc_scatter<<<(unsigned)((e + T - 1) / T), T, 0, st>>>(s);
        gp_cc_pair_scan<<<1, 1024, 0, st>>>(s, pairs, n_pairs, pref, po);
        pi.s = s;
        // The number of pairs is only known on the device; chunks beyond it return at once.  One chunk unless the pairs
        // times the multi-segment buckets exceed kCapSlotEntries (100 000 pairs over 50 000 nodes: 2.4 million slots, two).
        for (int32_t p0 = 0; p0 < Q; p0 += pairs_per_chunk) {
            pi.p0 = p0; pi.p1 = (int32_t)std::min<int64_t>((int64_t)p0 + pairs_per_chunk, Q);
            if (e > (size_t)kCapSeg) gp_cc_clear<<<(unsigned)std::min<size_t>((A + T - 1) / T, (size_t)c->sm_count * 16), T, 0, st>>>(pi);
            gp_cc_pass<<<pass_blocks, kCapThreads, 0, st>>>(pi);
        }
    }
    uint8_t* d_out = (uint8_t*)(b + o_out);
    if (Q > 0) gp_cc_decide<<<(unsigned)((q + T - 1) / T), T, 0, st>>>(Q, ai.count, app_pair, pairs, po, (int32_t)packer, d_out);
    GP_CUDA(c, cudaGetLastError());
    int herr = 0, aerr = 0;
    std::vector<int32_t> n_error(aff ? (size_t)G : 0);
    if (Q > 0) GP_CUDA(c, cudaMemcpyAsync(exceeds, d_out, q, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(&herr, s.err, 4, cudaMemcpyDeviceToHost, st));
    if (aff) {
        GP_CUDA(c, cudaMemcpyAsync(&aerr, b + as.o_err, 4, cudaMemcpyDeviceToHost, st));
        if (G > 0) GP_CUDA(c, cudaMemcpyAsync(n_error.data(), b + as.o_ne, 4 * (size_t)G, cudaMemcpyDeviceToHost, st));
    }
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (aff) { const gp_status ls = as.label_error(c, aerr, who); if (ls != GP_OK) return ls; }
    if (herr & kCcErrNegative) return bad(GP_ERR_INVALID, "negative resource request or exe_count");
    if (herr & kCcErrGroup) return bad(GP_ERR_INVALID, aff ? "driver group out of range (0..n_aff-1)" : "driver group out of range (-1 or 0..n_groups-1)");
    if (herr & kCcErrZone) return bad(GP_ERR_INVALID, "zone_id out of range");
    if (herr & kCcErrNodeGroup) return bad(GP_ERR_INVALID, "node_group out of range (-1 or 0..n_groups-1)");
    if (herr & kCcErrUnrepresentable) return bad(GP_ERR_UNREPRESENTABLE, "request >= 2^61");
    if (herr & kCcErrNodeQuantity) return bad(GP_ERR_UNREPRESENTABLE, "|allocatable| or |overhead| >= 2^61");
    if (aff && affinity_error)
        for (int32_t i = 0; i < Q; ++i) affinity_error[i] = n_error[a->group[i]] > 0 ? 1 : 0;
    return GP_OK;
}

extern "C" {

// DoesPodExceedClusterCapacity for a batch of stale drivers, any packer (EXT/unschedulablepods.go:132-166); see
// gangpack_capacity.cuh and DESIGN §2.2
gp_status gp_exceeds_cluster_capacity(gp_ctx* c, const gp_capacity_nodes* nodes, const gp_apps* a, gp_binpacker packer, uint8_t* exceeds) {
    if (!c) return GP_ERR_INVALID;
    return capacity_run(c, "gp_exceeds_cluster_capacity", nodes, nullptr, nullptr, a, packer, exceeds, nullptr);
}

// the same over the nodes each driver's required affinity matches (gangpack_affinity.cuh), overlapping sets allowed
gp_status gp_exceeds_cluster_capacity_affinity(gp_ctx* c, const gp_capacity_nodes* nodes, const gp_node_labels* labels,
                                               const gp_node_affinities* affinities, const gp_apps* a, gp_binpacker packer,
                                               uint8_t* exceeds, uint8_t* affinity_error) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_exceeds_cluster_capacity_affinity";
    if (!affinities) return fail(c, GP_ERR_INVALID, std::string(who) + ": missing arrays or negative sizes");
    return capacity_run(c, who, nodes, labels, affinities, a, packer, exceeds, affinity_error);
}

// GetRequiredNodeAffinity(...).Match for every (affinity, node); see gangpack_affinity.cuh
gp_status gp_match_node_affinity(gp_ctx* c, const gp_node_labels* labels, const gp_node_affinities* affinities, gp_affinity_match* out) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_match_node_affinity";
    gp_status s = check_affinity(c, labels, affinities, who);
    if (s != GP_OK) return s;
    if (!out) return fail(c, GP_ERR_INVALID, std::string(who) + ": missing arrays or negative sizes");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    Arena ar{c->capprep};
    AffStage as{};
    as.take(ar, labels, affinities);
    const size_t mbytes = 4 * (size_t)as.A * (size_t)as.words;
    const size_t o_member = ar.take(mbytes);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    GP_CUDA(c, as.upload(ar, labels, affinities, st));
    as.match(ar, (uint32_t*)(b + o_member), 0, as.A, st);
    GP_CUDA(c, cudaGetLastError());
    int aerr = 0;
    if (out->member && mbytes) GP_CUDA(c, cudaMemcpyAsync(out->member, b + o_member, mbytes, cudaMemcpyDeviceToHost, st));
    if (out->n_match && as.A) GP_CUDA(c, cudaMemcpyAsync(out->n_match, b + as.o_nm, 4 * (size_t)as.A, cudaMemcpyDeviceToHost, st));
    if (out->n_error && as.A) GP_CUDA(c, cudaMemcpyAsync(out->n_error, b + as.o_ne, 4 * (size_t)as.A, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaMemcpyAsync(&aerr, b + as.o_err, 4, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    return as.label_error(c, aerr, who);
}

// the failover reconciler's findNodes loop for a batch of stale drivers (EXT/failover.go:43-82, 286-436); see
// gangpack_reconcile.cuh and DESIGN §2.3
gp_status gp_reconcile_find_nodes(gp_ctx* c, const gp_usage_input* usage, const gp_reconcile_nodes* nodes, const gp_apps* a,
                                  gp_reconcile_results* out) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_reconcile_find_nodes";
    auto bad = [&](gp_status st, const char* what) { return fail(c, st, std::string(who) + ": " + what); };
    gp_status s = check_usage(c, usage, who);
    if (s != GP_OK) return s;
    if (!nodes || !a || !out || nodes->n_groups < 1 || a->n_apps < 0 || (usage->n_nodes > 0 && (!nodes->node_group || !nodes->creation)) ||
        (a->n_apps > 0 && (!a->exe_cpu_milli || !a->exe_mem_bytes || !a->exe_count || !out->placed)))
        return bad(GP_ERR_INVALID, "missing arrays or bad sizes (n_groups >= 1)");
    const int32_t n = usage->n_nodes, q = a->n_apps, G = nodes->n_groups;
    for (int32_t i = 0; i < n; ++i)
        if (nodes->node_group[i] < 0 || nodes->node_group[i] >= G) return bad(GP_ERR_INVALID, "node_group out of range");
    if ((s = check_requests(c, q, a->exe_cpu_milli, a->exe_mem_bytes, a->exe_gpu, who)) != GP_OK) return s;
    int64_t total = 0;
    for (int32_t i = 0; i < q; ++i) {
        const int32_t k = a->exe_count[i];
        if (k < 0) return bad(GP_ERR_INVALID, "negative exe_count");
        if (k > kMaxCount) return bad(GP_ERR_UNREPRESENTABLE, "exe_count > 2^24");
        if (a->group && (a->group[i] < 0 || a->group[i] >= G)) return bad(GP_ERR_INVALID, "instance group out of range");
        if (a->exec_out_off && a->exec_out_off[i] != total) return bad(GP_ERR_INVALID, "exec_out_off is not the prefix sum of exe_count");
        total += k;
    }
    if (a->exec_out_off && a->exec_out_off[q] != total) return bad(GP_ERR_INVALID, "exec_out_off is not the prefix sum of exe_count");
    if (total > 0 && (!out->executor_nodes || out->executor_nodes_cap < total))
        return bad(GP_ERR_CAPACITY, "executor_nodes_cap below the sum of exe_count");
    const bool want_avail = out->avail_cpu_milli || out->avail_mem_bytes || out->avail_gpu;
    if (n == 0) {                                       // every group is missing from orderedNodes
        for (int32_t i = 0; i < q; ++i) out->placed[i] = -1;
        return GP_OK;
    }
    if (q == 0 && !want_avail) return GP_OK;
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    long long *d_avail = nullptr, *d_sched = nullptr;   // usagebuf: scratch of the availability stage, charged in place below
    s = stage_availability(c, usage, st, &d_avail, &d_sched);
    if (s != GP_OK) return s;
    const size_t N = (size_t)n, Q = (size_t)q, Gs = (size_t)G, E = (size_t)total;
    Arena ar{c->reconbuf};
    const size_t o_grp = ar.take(4 * N), o_cre = ar.take(8 * N), o_fu = ar.take(N), o_fr = ar.take(N), o_keys = ar.take(sizeof(ReconKey) * N),
                 o_sorted = ar.take(sizeof(ReconKey) * N), o_pos = ar.take(4 * N), o_order = ar.take(4 * N), o_ngrp = ar.take(4 * N),
                 o_noff = ar.take(4 * (Gs + 1)), o_aoff = ar.take(4 * (Gs + 1)), o_exe = ar.take(24 * Q), o_cnt = ar.take(4 * Q),
                 o_agrp = ar.take(4 * Q), o_off = ar.take(8 * Q), o_list = ar.take(4 * Q), o_lk = ar.take(sizeof(LabelKey) * Q),
                 o_lks = ar.take(sizeof(LabelKey) * Q), o_apos = ar.take(4 * Q), o_apps = ar.take(4 * Q), o_placed = ar.take(4 * Q),
                 o_exn = ar.take(4 * E), o_word = ar.take(16);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    GP_CUDA(c, ar.upload(o_grp, nodes->node_group, 4 * N, st));
    GP_CUDA(c, ar.upload(o_cre, nodes->creation, 8 * N, st));
    if (nodes->unschedulable) GP_CUDA(c, ar.upload(o_fu, nodes->unschedulable, N, st));
    if (nodes->ready) GP_CUDA(c, ar.upload(o_fr, nodes->ready, N, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_word, 0, 16, st));  // claim counter, error word
    if (!c->recon_attr_set) {
        GP_CUDA(c, cudaFuncSetAttribute(gp_sort_tiles<ReconKey>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSortTile * sizeof(ReconKey))));
        c->recon_attr_set = true;
    }
    const int T = 256;
    const int nb = (n + T - 1) / T;
    ReconKey* keys = (ReconKey*)(b + o_keys);
    int32_t* pos = (int32_t*)(b + o_pos);
    int32_t* order = (int32_t*)(b + o_order);
    int32_t* ngrp = (int32_t*)(b + o_ngrp);
    gp_rc_node_keys<<<nb, T, 0, st>>>(n, G, (const int32_t*)(b + o_grp), (const long long*)(b + o_cre),
                                      nodes->unschedulable ? (const uint8_t*)(b + o_fu) : nullptr, nodes->ready ? (const uint8_t*)(b + o_fr) : nullptr,
                                      keys, ngrp);
    gp_sort_tiles<ReconKey><<<(n + kSortTile - 1) / kSortTile, kSortThreads, kSortTile * sizeof(ReconKey), st>>>(n, nullptr, keys, (ReconKey*)(b + o_sorted));
    gp_rank_by_search<ReconKey><<<nb, T, 0, st>>>(n, nullptr, keys, (const ReconKey*)(b + o_sorted), pos);
    gp_scatter_order<<<nb, T, 0, st>>>(n, pos, order);
    int32_t* apps = (int32_t*)(b + o_apps);
    int32_t* agrp = (int32_t*)(b + o_agrp);
    int32_t* cnt = (int32_t*)(b + o_word + 8);
    if (q > 0) {
        // exe cpu, mem, gpu columns, counts, groups and offsets
        GP_CUDA(c, ar.upload(o_exe, a->exe_cpu_milli, 8 * Q, st));
        GP_CUDA(c, ar.upload(o_exe + 8 * Q, a->exe_mem_bytes, 8 * Q, st));
        if (a->exe_gpu) GP_CUDA(c, ar.upload(o_exe + 16 * Q, a->exe_gpu, 8 * Q, st));
        else GP_CUDA(c, cudaMemsetAsync(b + o_exe + 16 * Q, 0, 8 * Q, st));
        GP_CUDA(c, ar.upload(o_cnt, a->exe_count, 4 * Q, st));
        if (a->group) GP_CUDA(c, ar.upload(o_agrp, a->group, 4 * Q, st));
        else GP_CUDA(c, cudaMemsetAsync(agrp, 0, 4 * Q, st));
        if (a->exec_out_off) GP_CUDA(c, ar.upload(o_off, a->exec_out_off, 8 * Q, st));
        else {
            std::vector<int64_t>& off = c->host_off;
            off.resize(Q);
            int64_t run = 0;
            for (int32_t i = 0; i < q; ++i) { off[i] = run; run += a->exe_count[i]; }
            GP_CUDA(c, ar.upload(o_off, off.data(), 8 * Q, st));
        }
        // the stale drivers partitioned by group, call order kept inside each group
        const int qb = (q + T - 1) / T;
        gp_rc_app_list<<<qb, T, 0, st>>>(q, (int32_t*)(b + o_list), cnt);
        launch_label_resort(q, cnt, (const int32_t*)(b + o_list), agrp, (LabelKey*)(b + o_lk), (LabelKey*)(b + o_lks), (int32_t*)(b + o_apos),
                            apps, st);
    }
    gp_rc_offsets<<<(unsigned)((Gs + T) / T), T, 0, st>>>(G, n, order, ngrp, q, apps, agrp, (int32_t*)(b + o_noff), (int32_t*)(b + o_aoff));
    if (q > 0) {
        RcLoopIn li{};
        li.avail = d_avail; li.order = order; li.noff = (const int32_t*)(b + o_noff);
        li.apps = apps; li.aoff = (const int32_t*)(b + o_aoff);
        li.exe = (const long long*)(b + o_exe); li.count = (const int32_t*)(b + o_cnt); li.out_off = (const long long*)(b + o_off);
        li.placed = (int32_t*)(b + o_placed); li.exec_nodes = (int32_t*)(b + o_exn);
        li.claim = (unsigned int*)(b + o_word); li.err = (int*)(b + o_word + 4);
        li.n = n; li.q = q; li.n_groups = G;
        // one CTA per instance group; CTAs that find no group left return at once
        const int blocks = (int)std::min<int64_t>(G, (int64_t)c->sm_count * 8);
        gp_rc_loop<<<blocks, kRcThreads, 0, st>>>(li);
    }
    GP_CUDA(c, cudaGetLastError());
    int herr = 0;
    if (q > 0) {
        GP_CUDA(c, cudaMemcpyAsync(out->placed, b + o_placed, 4 * Q, cudaMemcpyDeviceToHost, st));
        if (E) GP_CUDA(c, cudaMemcpyAsync(out->executor_nodes, b + o_exn, 4 * E, cudaMemcpyDeviceToHost, st));
        GP_CUDA(c, cudaMemcpyAsync(&herr, b + o_word + 4, 4, cudaMemcpyDeviceToHost, st));
    }
    int64_t* outs[3] = {out->avail_cpu_milli, out->avail_mem_bytes, out->avail_gpu};
    for (int d = 0; d < 3; ++d)
        if (outs[d]) GP_CUDA(c, cudaMemcpyAsync(outs[d], d_avail + N * (size_t)d, 8 * N, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    if (herr & kRcErrDomain) return bad(GP_ERR_UNREPRESENTABLE, "an availability the loop charged lies outside the exact-int64 domain (|v| >= 2^61)");
    return GP_OK;
}

// The overhead computer's per-call side (EXT/overhead.go:105-153) for a list of nodes; see gangpack_overhead.cuh
gp_status gp_node_overhead(gp_ctx* c, const gp_overhead_pods* p, const gp_overhead_reservations* r, int32_t n_nodes,
                           const int32_t* node_ids, gp_overhead_out* out) {
    if (!c) return GP_ERR_INVALID;
    static const char* who = "gp_node_overhead";
    auto bad = [&](gp_status st, const char* what) { return fail(c, st, std::string(who) + ": " + what); };
    if (!p || !r || !out || p->n_pods < 0 || p->n_node_ids < 0 || p->n_app_keys < 0 || p->n_app_ids < 0 || p->n_names < 0 ||
        r->n_rr < 0 || r->n_soft < 0 || n_nodes < 0 || (n_nodes > 0 && !node_ids) ||
        (p->n_pods > 0 && (!p->node_id || !p->req_cpu_milli || !p->req_mem_bytes || !p->app_key || !p->app_id || !p->name_id)) ||
        (r->n_rr > 0 && (!r->rr_app_key || !r->rr_pod_off)) || (r->n_soft > 0 && (!r->soft_app_id || !r->soft_pod_off)))
        return bad(GP_ERR_INVALID, "missing arrays or negative sizes");
    if (p->n_pods > INT32_MAX) return bad(GP_ERR_INVALID, "n_pods must be below 2^31");
    // CSR offsets (one per reservation: host-sized); the entries themselves are checked on the device
    auto entries = [](const int64_t* off, int32_t n, int64_t* total) {
        if (n == 0) { *total = 0; return !off || off[0] == 0; }
        if (off[0] != 0) return false;
        for (int32_t i = 0; i < n; ++i) if (off[i + 1] < off[i]) return false;
        *total = off[n];
        return true;
    };
    int64_t er = 0, es = 0;
    if (!entries(r->rr_pod_off, r->n_rr, &er) || !entries(r->soft_pod_off, r->n_soft, &es))
        return bad(GP_ERR_INVALID, "rr_pod_off or soft_pod_off does not start at 0 or decreases");
    if ((er > 0 && !r->rr_pod_name) || (es > 0 && !r->soft_pod_name)) return bad(GP_ERR_INVALID, "missing arrays or negative sizes");
    if (er + es > ((int64_t)1 << 30)) return bad(GP_ERR_INVALID, "more than 2^30 reservation entries");
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    const size_t P = (size_t)p->n_pods, N = (size_t)n_nodes, R = (size_t)r->n_rr, S = (size_t)r->n_soft;
    size_t H = 64;
    while (H < 2 * (size_t)(er + es)) H <<= 1;           // at most half full: every probe ends
    Arena ar{c->overbuf};
    const size_t o_node = ar.take(4 * P), o_req = ar.take(24 * P), o_listed = ar.take(P), o_ak = ar.take(4 * P), o_ai = ar.take(4 * P),
                 o_name = ar.take(4 * P), o_exe = ar.take(P), o_spark = ar.take(P), o_has = ar.take(P),
                 o_rkey = ar.take(4 * R), o_roff = ar.take(8 * (R + 1)), o_rname = ar.take(4 * (size_t)er),
                 o_skey = ar.take(4 * S), o_soff = ar.take(8 * (S + 1)), o_sname = ar.take(4 * (size_t)es), o_qn = ar.take(4 * N),
                 o_rok = ar.take(4 * (size_t)p->n_app_keys), o_soa = ar.take(4 * (size_t)p->n_app_ids),
                 o_ron = ar.take(4 * (size_t)p->n_node_ids), o_set = ar.take(8 * H),
                 o_acc = ar.take(96 * N), o_word = ar.take(16), o_out = ar.take(48 * N);
    GP_CUDA(c, ar.reserve());
    char* b = ar.base();
    // the directories and the hash set start at -1 / empty; the sums, n_warned and the error word at 0
    GP_CUDA(c, cudaMemsetAsync(b + o_rok, 0xff, o_set + 8 * H - o_rok, st));
    GP_CUDA(c, cudaMemsetAsync(b + o_acc, 0, o_word + 16 - o_acc, st));
    struct Piece { size_t o; const void* src; size_t bytes; };
    const Piece pieces[] = {
        {o_node, p->node_id, 4 * P}, {o_req, p->req_cpu_milli, 8 * P}, {o_req + 8 * P, p->req_mem_bytes, 8 * P},
        {o_req + 16 * P, p->req_gpu, 8 * P}, {o_listed, p->listed, P}, {o_ak, p->app_key, 4 * P}, {o_ai, p->app_id, 4 * P},
        {o_name, p->name_id, 4 * P}, {o_exe, p->is_executor, P}, {o_spark, p->spark_scheduler, P},
        {o_rkey, r->rr_app_key, 4 * R}, {o_roff, r->rr_pod_off, R ? 8 * (R + 1) : 0}, {o_rname, r->rr_pod_name, 4 * (size_t)er},
        {o_skey, r->soft_app_id, 4 * S}, {o_soff, r->soft_pod_off, S ? 8 * (S + 1) : 0}, {o_sname, r->soft_pod_name, 4 * (size_t)es},
        {o_qn, node_ids, 4 * N}};
    for (const Piece& pc : pieces)
        if (pc.src && pc.bytes) GP_CUDA(c, ar.upload(pc.o, pc.src, pc.bytes, st));
    OhMaps M{(int32_t*)(b + o_rok), (int32_t*)(b + o_soa), (int32_t*)(b + o_ron), (unsigned long long*)(b + o_set), (uint32_t)(H - 1),
             r->n_rr};
    int* d_err = (int*)(b + o_word + 8);
    const int T = 256, cap = c->sm_count * 8;
    const long long n_dir = (long long)R + (long long)S + (long long)N;
    if (n_dir > 0) {
        OhDirIn D{r->n_rr, r->n_soft, n_nodes, p->n_app_keys, p->n_app_ids, p->n_node_ids,
                  (const int32_t*)(b + o_rkey), (const int32_t*)(b + o_skey), (const int32_t*)(b + o_qn)};
        gp_oh_dir<<<(unsigned)std::min<long long>((n_dir + T - 1) / T, cap), T, 0, st>>>(D, M, d_err);
    }
    if (er + es > 0) {
        OhSetIn si{(const long long*)(b + o_roff), (const int32_t*)(b + o_rname), (const long long*)(b + o_soff),
                   (const int32_t*)(b + o_sname), r->n_rr, r->n_soft, p->n_names, (long long)er, (long long)es};
        gp_oh_insert<<<(unsigned)std::min<long long>((er + es + T - 1) / T, cap), T, 0, st>>>(si, M, d_err);
    }
    OhAcc A{(unsigned long long*)(b + o_acc), (unsigned long long*)(b + o_word), n_nodes};
    if (P > 0) {
        OhPodsIn pi{};
        pi.n = (long long)P; pi.n_node_ids = p->n_node_ids; pi.n_app_keys = p->n_app_keys; pi.n_app_ids = p->n_app_ids; pi.n_names = p->n_names;
        pi.node_id = (const int32_t*)(b + o_node);
        for (int d = 0; d < 3; ++d) pi.req[d] = (d < 2 || p->req_gpu) ? (const long long*)(b + o_req) + P * (size_t)d : nullptr;
        pi.listed = p->listed ? (const uint8_t*)(b + o_listed) : nullptr;
        pi.app_key = (const int32_t*)(b + o_ak); pi.app_id = (const int32_t*)(b + o_ai); pi.name_id = (const int32_t*)(b + o_name);
        pi.is_executor = p->is_executor ? (const uint8_t*)(b + o_exe) : nullptr;
        pi.spark_scheduler = p->spark_scheduler ? (const uint8_t*)(b + o_spark) : nullptr;
        pi.has_reservation = (uint8_t*)(b + o_has);
        gp_oh_pods<<<(unsigned)((P + kOhThreads - 1) / kOhThreads), kOhThreads, 0, st>>>(pi, M, A, d_err);
    }
    long long* d_out = (long long*)(b + o_out);
    if (N > 0) gp_oh_finish<<<(unsigned)((N + T - 1) / T), T, 0, st>>>(A, d_out, d_err);
    GP_CUDA(c, cudaGetLastError());
    int64_t* outs[6] = {out->overhead_cpu_milli, out->overhead_mem_bytes, out->overhead_gpu,
                        out->nonsched_cpu_milli, out->nonsched_mem_bytes, out->nonsched_gpu};
    for (int k = 0; k < 6; ++k)
        if (outs[k] && N) GP_CUDA(c, cudaMemcpyAsync(outs[k], d_out + N * (size_t)k, 8 * N, cudaMemcpyDeviceToHost, st));
    if (out->has_reservation && P) GP_CUDA(c, cudaMemcpyAsync(out->has_reservation, b + o_has, P, cudaMemcpyDeviceToHost, st));
    unsigned long long word[2] = {0, 0};                 // n_warned, error bits
    GP_CUDA(c, cudaMemcpyAsync(word, b + o_word, 16, cudaMemcpyDeviceToHost, st));
    GP_CUDA(c, cudaStreamSynchronize(st));
    const int herr = (int)word[1];
    if (herr & kOhErrRange) return bad(GP_ERR_INVALID, "an id out of its range (node, app key, app id, name or query node)");
    if (herr & kOhErrAppPair) return bad(GP_ERR_INVALID, "app_key and app_id disagree on -1");
    if (herr & kOhErrDuplicate) return bad(GP_ERR_INVALID, "a query node id, rr_app_key or soft_app_id given twice");
    if (herr & kOhErrNegative) return bad(GP_ERR_INVALID, "negative request");
    if (herr & kOhErrRequest) return bad(GP_ERR_UNREPRESENTABLE, "request >= 2^61");
    if (herr & kOhErrSum) return bad(GP_ERR_UNREPRESENTABLE, "a per-node sum >= 2^61");
    if (out->n_warned) *out->n_warned = (int64_t)word[0];
    return GP_OK;
}

}  // extern "C"

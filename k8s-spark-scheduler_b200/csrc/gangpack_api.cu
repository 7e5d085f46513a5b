// gangpack_api.cu -- the context and the snapshot: the slot-layout kernels, gp_create .. gp_synchronize, gp_set_snapshot,
// gp_set_snapshot_device and gp_get_snapshot.  The other entry points of include/gangpack.h live in gangpack_pack.cu,
// gangpack_zones.cu, gangpack_cluster.cu, gangpack_marker.cu and gangpack_multi.cu.
// There is no CPU code path in this library: without a usable CUDA device gp_create fails.
#include "gangpack_ctx.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

// =============================================================================================
// kernels
// =============================================================================================

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
// K2 gp_build_slots_drv: every CTA first folds K1's parts (visible once its pdl_wait has returned: no fence or counter
//    needed) into the maxima its compact views shift by; CTA 0 publishes them in SnapMeta (flags, max_avail,
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
    pdl_trigger();                       // K2 may start: it waits for this launch before it reads anything of it
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

// seg_pre[g] = table segments (gangpack_tables.cuh) of the groups before g, max(1, ceil(ne / kTabSeg)) each: an empty group
// still has the one segment that writes its total and first_host; seg_pre[n_groups] = all of them.  Called by a whole CTA.
__device__ __forceinline__ void segment_prefix(int32_t n_groups, const int32_t* __restrict__ exec_off, int32_t* __restrict__ seg_pre) {
    __shared__ uint32_t part[kSnapThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t carry = 0;
    for (int32_t g0 = 0; g0 < n_groups; g0 += kSnapThreads) {
        const int32_t g = g0 + (int32_t)threadIdx.x;
        const uint32_t n = g < n_groups ? (uint32_t)max(1, (exec_off[g + 1] - exec_off[g] + kTabSeg - 1) / kTabSeg) : 0u;
        const uint32_t incl = warp_incl_scan(n, lane);
        if (lane == 31) part[w] = incl;
        __syncthreads();
        uint32_t before = carry, all = carry;
        for (int t = 0; t < kSnapThreads / 32; ++t) { if (t < w) before += part[t]; all += part[t]; }
        if (g < n_groups) seg_pre[g] = (int32_t)(before + incl - n);
        carry = all;
        __syncthreads();
    }
    if (threadIdx.x == 0) seg_pre[n_groups] = (int32_t)carry;
}

// Launched as K1's dependent: it may start once every CTA of K1 has started, and waits for K1 to end (pdl_wait) before it
// reads anything K1 writes.  Its last CTA first writes the snapshot's segment prefix, which gp_decide_tables reads after
// the layout; it reads only exec_off, an input of the layout, complete before K1 started.
__global__ void __launch_bounds__(kSnapThreads) gp_build_slots_drv(int32_t n_slots, int32_t n_groups, int32_t n_nodes, int32_t n_drv,
                                   const int32_t* __restrict__ exec_off, const int32_t* __restrict__ drv_off,
                                   const int32_t* __restrict__ drv_order, const int32_t* __restrict__ drv_pos,
                                   const int64_t* __restrict__ cpu, const int64_t* __restrict__ mem, const int64_t* __restrict__ gpu,
                                   longlong2* __restrict__ pair, int64_t* __restrict__ sgpu, int32_t* __restrict__ slot_node,
                                   int32_t* __restrict__ node_slot, int32_t* __restrict__ drv_slot, const SnapPart* __restrict__ parts,
                                   int32_t n_parts, SnapMeta* __restrict__ meta, uint2* __restrict__ pair32,
                                   int32_t* __restrict__ seg_pre) {
    __shared__ long long s_max[2];
    pdl_trigger();                       // a pack call's gp_decide_tables may start: it waits for this launch (see there)
    if (blockIdx.x == gridDim.x - 1) segment_prefix(n_groups, exec_off, seg_pre);
    pdl_wait();
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

// Device-visible alias of a host buffer, or nullptr.  Buffers from gp_alloc_pinned are known; anything
// else is asked of the driver (cudaHostRegister / cudaHostAlloc memory of the caller qualifies).
const void* mapped_ptr(gp_ctx* c, const void* p, size_t bytes) {
    if (!p || !c->zero_copy) return nullptr;
    const char* q = static_cast<const char*>(p);
    for (const auto& b : c->pinned_blocks)
        if (q >= b.first && q + bytes <= b.first + b.second) return p;     // UVA: same address on the device
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (a.type == cudaMemoryTypeHost && a.devicePointer) return a.devicePointer;
    return nullptr;
}

gp_status fail(gp_ctx* ctx, gp_status st, const std::string& msg) {
    ctx->err = msg;
    return st;
}

Snapshot make_snapshot(const gp_ctx* c) {
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

// ---- snapshot ---------------------------------------------------------------------------------

// Build the slot layout from DEVICE-resident gp_nodes arrays on `st`.  copy_nodes: the layout kernel also copies the node
// table into node_cpu / node_mem / node_gpu (reserved by the caller; false when dn already points at them).
gp_status build_snapshot_device(gp_ctx* c, const gp_nodes* dn, int32_t n_exec, int32_t n_drv, cudaStream_t st,
                                bool copy_nodes) {
    const int32_t n_slots = n_exec + n_drv;
    GP_CUDA(c, c->pair.reserve(sizeof(longlong2) * (size_t)(n_slots + 1)));
    GP_CUDA(c, c->pair32.reserve(sizeof(uint2) * (size_t)(n_slots + 1)));
    GP_CUDA(c, c->sgpu.reserve(sizeof(int64_t) * (size_t)(n_slots + 1)));
    GP_CUDA(c, c->slot_node.reserve(sizeof(int32_t) * (size_t)(n_slots + 1)));
    GP_CUDA(c, c->node_slot.reserve(sizeof(int32_t) * (size_t)(dn->n_nodes + 1)));
    GP_CUDA(c, c->drv_slot.reserve(sizeof(int32_t) * (size_t)(n_drv + 1)));
    GP_CUDA(c, c->groups.reserve(sizeof(GroupDesc) * (size_t)dn->n_groups));
    GP_CUDA(c, c->drv_pos.reserve(sizeof(int32_t) * (size_t)(dn->n_nodes + 1)));
    GP_CUDA(c, c->seg_pre.reserve(sizeof(int32_t) * (size_t)(dn->n_groups + 1)));
    int64_t* node_cpu = copy_nodes ? c->node_cpu.as<int64_t>() : nullptr;
    const int T = kSnapThreads;
    const int32_t n1 = std::max(std::max(std::max(n_exec, n_drv), dn->n_groups), node_cpu ? dn->n_nodes : 0);
    const int32_t blocks1 = (n1 + T - 1) / T;
    GP_CUDA(c, c->snap_part.reserve(sizeof(SnapPart) * (size_t)blocks1));
    SnapPart* parts = c->snap_part.as<SnapPart>();
    struct { gp_nodes dn; int32_t n_exec, n_drv; void* buf[14]; } key{};
    key.dn = *dn; key.n_exec = n_exec; key.n_drv = n_drv;
    void* bufs[14] = {c->pair.p, c->pair32.p, c->sgpu.p, c->slot_node.p, c->node_slot.p, c->drv_slot.p, c->groups.p, c->snap_flags.p,
                      node_cpu, c->node_mem.p, c->node_gpu.p, c->drv_pos.p, c->snap_part.p, c->seg_pre.p};
    std::memcpy(key.buf, bufs, sizeof(bufs));
    gp_status rs = run_cached(c, c->g_snapshot, &key, sizeof(key), st, [&](int& launches) -> gp_status {
        gp_build_slots_exec<<<blocks1, T, 0, st>>>(
            n_exec, n_drv, dn->n_groups, dn->n_nodes, dn->exec_off, dn->drv_off, dn->exec_order, dn->drv_order, dn->avail_cpu_milli,
            dn->avail_mem_bytes, dn->avail_gpu, c->groups.as<GroupDesc>(), c->pair.as<longlong2>(), c->sgpu.as<int64_t>(),
            c->slot_node.as<int32_t>(), c->node_slot.as<int32_t>(), c->drv_pos.as<int32_t>(), parts, node_cpu,
            c->node_mem.as<int64_t>(), c->node_gpu.as<int64_t>());
        // threads [0, n_slots]: slots; [n_slots + 1, n_slots + 1 + n_nodes]: nodes
        GP_CUDA(c, launch_pdl(true, (n_slots + dn->n_nodes + 1 + T) / T, T, st, gp_build_slots_drv,
            n_slots, dn->n_groups, dn->n_nodes, n_drv, dn->exec_off, dn->drv_off, dn->drv_order, c->drv_pos.as<int32_t>(),
            dn->avail_cpu_milli, dn->avail_mem_bytes, dn->avail_gpu, c->pair.as<longlong2>(), c->sgpu.as<int64_t>(),
            c->slot_node.as<int32_t>(), c->node_slot.as<int32_t>(), c->drv_slot.as<int32_t>(), parts, blocks1,
            c->snap_flags.as<SnapMeta>(), c->pair32.as<uint2>(), c->seg_pre.as<int32_t>()));
        GP_CUDA(c, cudaGetLastError());
        launches = 0;       // (the snapshot layout is not part of a pack call's launch count)
        return GP_OK;
    });
    if (rs != GP_OK) return rs;
    c->n_nodes = dn->n_nodes; c->n_groups = dn->n_groups; c->n_exec = n_exec; c->n_drv = n_drv; c->n_slots = n_slots;
    return GP_OK;
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

gp_status gp_set_snapshot(gp_ctx* c, const gp_nodes* n) {
    if (!enter(c)) return GP_ERR_INVALID;
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
        c->held.host_copy_overwritten();
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
    c->held.commit();
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
    GP_TRY(build_snapshot_device(c, &dn, n_exec, n_drv, st));
    c->held.laid_out_snapshot();
    // GP_CFG_ASYNC_SNAPSHOT with page-locked inputs: return while the device is still reading them -- the upload and the
    // slot layout then overlap the H2D copies of the gp_pack_* call that follows
    if (!(c->async_snapshot && all_mapped)) GP_CUDA(c, cudaStreamSynchronize(st));   // the caller may reuse its host buffers
    return GP_OK;
}

gp_status gp_set_snapshot_device(gp_ctx* c, const gp_nodes* dn, int32_t n_exec, int32_t n_drv, void* stream) {
    if (!enter(c)) return GP_ERR_INVALID;
    if (!dn || dn->n_nodes < 0 || dn->n_groups < 1 || !dn->exec_off || !dn->drv_off || n_exec < 0 || n_drv < 0 ||
        (n_exec > 0 && !dn->exec_order) || (n_drv > 0 && !dn->drv_order))
        return fail(c, GP_ERR_INVALID, "gp_set_snapshot_device: missing arrays or bad sizes");
    c->held.commit();
    GP_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream;
    // keep a node-table copy so gp_get_snapshot can answer for nodes outside every group: the layout kernel makes it
    const size_t nb = sizeof(int64_t) * (size_t)(dn->n_nodes + 1);
    GP_CUDA(c, c->node_cpu.reserve(nb)); GP_CUDA(c, c->node_mem.reserve(nb)); GP_CUDA(c, c->node_gpu.reserve(nb));
    GP_TRY(build_snapshot_device(c, dn, n_exec, n_drv, st, dn->n_nodes > 0));
    c->held.laid_out_device(c->async_snapshot ? st : nullptr);      // the layout is the last work on st
    return GP_OK;
}

gp_status gp_get_snapshot(gp_ctx* c, int64_t* cpu, int64_t* mem, int64_t* gpu) {
    if (!enter(c)) return GP_ERR_INVALID;
    GP_TRY(require(c, c->held.snapshot("no snapshot"), "gp_get_snapshot"));
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

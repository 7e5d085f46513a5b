// gangpack_fifo.cuh -- FIFO modes: fitEarlierDrivers (internal/extender/resource.go:224-262) on the device.
//
// The loop is a true sequential dependency inside one instance group (application i+1 sees the
// usage application i subtracted), so parallelism comes from WITHIN an application and ACROSS
// instance groups: one persistent CTA owns one group's queue.
//   * WARP FIRST: the typical application resolves inside the first few hundred live nodes, so warp 0 walks the queue
//     alone -- first fitting driver, 32 nodes per step from the live prefix, warp scan, emit, charge -- without a single
//     block-wide barrier.  The other warps sleep on a named hardware barrier (bar.sync 1) and are woken only when an
//     application outgrows the warp's window budget or needs the exact three-phase decision: then the whole CTA runs
//     fifo_app() below (1024 nodes per step).
//   * the group's executor-order slots (16 B (cpu,mem) records) are staged into shared memory with
//     TMA bulk copies (cp.async.bulk + mbarrier) and written back with a bulk store at the end, so the
//     block-serial commit of reservations never leaves the SM;
//   * every thread owns one node per step: block-wide reduction / prefix scan / first-feasible vote
//     replace the warp primitives of the independent kernel;
//   * slots that do not fit shared memory (very large groups, driver-only spare slots, the gpu
//     dimension) are served from global memory by the same accessors.
#pragma once

#include "gangpack_kernels.cuh"

namespace gp {

constexpr int kFifoThreads = 256;     // warp 0 does the common case alone and wants registers; the CTA path is the exception
constexpr int kFifoWarps = kFifoThreads / 32;
constexpr int kFifoSmemSlots = 11776;          // 184 KB of (cpu,mem) records
constexpr int kFifoCache = 12288;              // uint16 capacity cache entries (24 KB)

struct FifoScratch {
    unsigned long long bar;                    // mbarrier for the TMA staging
    uint32_t part_a[2][kFifoWarps];
    uint32_t part_b[2][kFifoWarps];
    int32_t found[2][kFifoWarps];
    unsigned mask[kFifoWarps];
    int32_t first_live_e;                      // executor-order positions before this are dead for the whole batch
    int32_t first_live_d;                      // same for driver-order entries
    int32_t cmd_app;                           // warp 0 -> helpers: application to run block-wide, -1 = exit
    uint32_t cmd_seq;
    int32_t list_base;                         // this group's slice of the per-group application lists
    int32_t result;                            // block path -> warp 0
};

// dead for every application of the batch (see GroupMin)
__device__ __forceinline__ bool dead_for(const long long* mn, longlong2 v, int64_t gpu_avail, bool use_gpu) {
    bool dead = v.x < mn[0] || v.y < mn[1] || v.x < 0 || v.y < 0;
    if (use_gpu) dead = dead || gpu_avail < mn[2] || gpu_avail < 0;
    return dead;
}

// ---- TMA 1-D bulk copies -----------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}

// ---- the group's mutable view: slots [0, n_smem) live in shared memory, the rest in global ------------
struct FifoView {
    longlong2* sp;          // shared-memory copy of slots [0, n_smem)
    longlong2* gp;          // global slots of this group (s.pair + sbase)
    int64_t* gg;            // global gpu values of this group
    int32_t n_smem;
    bool all_smem;          // every slot this kernel touches is staged (warp 0's fast accessors rely on it)
    __device__ __forceinline__ longlong2* pair_ptr(int32_t local) const { return local < n_smem ? sp + local : gp + local; }
    __device__ __forceinline__ longlong2 pair(int32_t local) const {
        if (local < n_smem) return sp[local];
        longlong2 v;
        asm volatile("ld.global.v2.s64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(gp + local) : "memory");
        return v;
    }
    __device__ __forceinline__ int64_t gpu(int32_t local) const {
        int64_t v;
        asm volatile("ld.global.s64 %0, [%1];" : "=l"(v) : "l"(gg + local) : "memory");
        return v;
    }
    __device__ __forceinline__ void charge(int32_t local, long long mult, int64_t cpu, int64_t mem, int64_t gpu_req) const {
        longlong2* pp = pair_ptr(local);
        longlong2 v = *pp;
        v.x -= mult * cpu; v.y -= mult * mem;
        *pp = v;
        if (gpu_req != 0) gg[local] -= mult * gpu_req;
    }
};

// the same view when EVERY slot the kernel touches is staged in shared memory (identical driver / executor orders, group
// within the staging area): no shared-or-global branch on warp 0's critical path
struct FifoViewS {
    longlong2* sp;
    int64_t* gg;
    __device__ __forceinline__ longlong2 pair(int32_t local) const { return sp[local]; }
    __device__ __forceinline__ int64_t gpu(int32_t local) const {
        int64_t v;
        asm volatile("ld.global.s64 %0, [%1];" : "=l"(v) : "l"(gg + local) : "memory");
        return v;
    }
    __device__ __forceinline__ void charge(int32_t local, long long mult, int64_t cpu, int64_t mem, int64_t gpu_req) const {
        longlong2 v = sp[local];
        v.x -= mult * cpu; v.y -= mult * mem;
        sp[local] = v;
        if (gpu_req != 0) gg[local] -= mult * gpu_req;
    }
};

// capacity of one slot for one application (fast or general class), clamped to k
template <bool FAST> struct FifoCaps;
template <> struct FifoCaps<true> : Caps<true> {
    template <class V>
    __device__ __forceinline__ uint32_t capr(const V& v, int32_t local, int64_t r_cpu, int64_t r_mem, int64_t r_gpu) const {
        longlong2 p = v.pair(local);
        uint32_t c = cap_pair(p, r_cpu, r_mem);
        if (use_gpu) c = min(c, fast_q(v.gpu(local) - r_gpu, gpu));
        return c;
    }
};
template <> struct FifoCaps<false> : Caps<false> {
    template <class V>
    __device__ __forceinline__ uint32_t capr(const V& v, int32_t local, int64_t r_cpu, int64_t r_mem, int64_t r_gpu) const {
        longlong2 p = v.pair(local);
        uint32_t c = min(cap_dim(p.x - r_cpu, cpu, k), cap_dim(p.y - r_mem, mem, k));
        if (use_gpu) c = min(c, cap_dim(v.gpu(local) - r_gpu, gpu, k));
        return c;
    }
};

// ---- block primitives (all 1024 threads call them; `buf` alternates so one barrier per call suffices)
__device__ __forceinline__ void block_reduce2(FifoScratch& sh, int& buf, uint32_t a, uint32_t b, uint32_t& ra, uint32_t& rb) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t wa = warp_sum(a), wb = warp_sum(b);
    if (lane == 0) { sh.part_a[buf][w] = wa; sh.part_b[buf][w] = wb; }
    __syncthreads();
    const int nw = blockDim.x >> 5;
    ra = warp_sum(lane < nw ? sh.part_a[buf][lane] : 0u);
    rb = warp_sum(lane < nw ? sh.part_b[buf][lane] : 0u);
    buf ^= 1;
}
__device__ __forceinline__ void block_excl_scan(FifoScratch& sh, int& buf, uint32_t v, uint32_t& excl, uint32_t& total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t incl = warp_incl_scan(v, lane);
    if (lane == 31) sh.part_a[buf][w] = incl;
    __syncthreads();
    uint32_t t = lane < (int)(blockDim.x >> 5) ? sh.part_a[buf][lane] : 0u;
    uint32_t ti = warp_incl_scan(t, lane);
    uint32_t before = __shfl_sync(kFull, ti - t, w);     // sum of the totals of the warps before mine
    total = __shfl_sync(kFull, ti, 31);
    excl = before + incl - v;
    buf ^= 1;
}
// value of the first thread (in thread order) whose predicate holds, or -1
__device__ __forceinline__ int32_t block_first(FifoScratch& sh, int& buf, bool pred, int32_t value) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned vote = __ballot_sync(kFull, pred);
    int32_t first = vote ? __shfl_sync(kFull, value, __ffs(vote) - 1) : -1;
    if (lane == 0) sh.found[buf][w] = first;
    __syncthreads();
    int32_t f = lane < (int)(blockDim.x >> 5) ? sh.found[buf][lane] : -1;
    unsigned v2 = __ballot_sync(kFull, f >= 0);
    int32_t r = v2 ? __shfl_sync(kFull, f, __ffs(v2) - 1) : -1;
    buf ^= 1;
    return r;
}

// ---- one application, the whole CTA ----------------------------------------------------------------
template <int ALGO, int FIFO_MODE, bool FAST>
__device__ __forceinline__ int32_t fifo_app(const Snapshot& s, const GroupDesc& g, const FifoView& view, const PrepApp* __restrict__ pa,
                                            int32_t* __restrict__ executor_nodes, int2* __restrict__ scratch,
                                            uint16_t* __restrict__ cache, FifoScratch& sh, int& buf, WarpStats& st,
                                            const GroupMin& gm, uint32_t app_seq) {
    const int tid = threadIdx.x, lane = tid & 31;
    const int32_t nt = (int32_t)blockDim.x;
    FifoCaps<FAST> a;
    a.init(pa, (pa->flags & kAppUsesGpu) || (s.meta->flags & kSnapGpuNegative));
    const uint32_t k = a.k;
    const uint32_t lmax = (uint32_t)pa->lmax;
    const int32_t ne = g.ne;
    const int64_t out_off = pa->out_off;
    int32_t* out = executor_nodes + out_off;
    int2* list = scratch ? scratch + out_off : nullptr;
    const int32_t* slot_node = s.slot_node + g.sbase;
    const bool cache_ok = k <= 0xFFFFu;

    const int32_t start_e = sh.first_live_e;      // block-uniform (written before the last barrier)
    const int32_t start_d = sh.first_live_d;

    // ---- optimistic single pass (tightly-pack): the first driver candidate that FITS is the reference's
    // answer whenever the executors fit with it (binpack.go:67-85), which is the common case.  Capacities are
    // evaluated once, ExecutorNodes is emitted on the fly, the charges are deferred until the placement is
    // known to be complete (the takes wait in the shared-memory cache).  If the executors do not fit with
    // that candidate nothing has been charged and the general three-phase path below decides exactly.
    if (ALGO == 0 && k != 0 && cache_ok) {
        const bool refresh = (app_seq & 3u) == 0;          // dead-prefix bookkeeping every 4th application
        int32_t j1 = -1;
        for (int32_t j0 = start_d; j0 < g.nd && j1 < 0; j0 += nt) {
            int32_t j = j0 + tid;
            bool fits = false, alive = false;
            if (j < g.nd) {
                const int32_t ls = s.drv_slot[g.dbase + j];
                longlong2 v = view.pair(ls);
                const int64_t gv = a.use_gpu ? view.gpu(ls) : 0;
                fits = !(a.d_cpu > v.x) && !(a.d_mem > v.y) && !(a.use_gpu && a.d_gpu > gv);
                alive = !dead_for(gm.drv, v, gv, a.use_gpu);
            }
            if (refresh && j0 == start_d) {
                int32_t f = block_first(sh, buf, alive, j);
                if (tid == 0) sh.first_live_d = f >= 0 ? f : (j0 + nt < g.nd ? j0 + nt : g.nd);
            }
            j1 = block_first(sh, buf, fits, j);
            if (tid == 0) st.drivers += (unsigned long long)((g.nd - j0) < nt ? (g.nd - j0) : nt);
        }
        if (j1 < 0) return -1;                               // no node can host the driver at all
        const int32_t d1 = s.drv_slot[g.dbase + j1];
        const uint32_t cd1 = d1 < ne ? a.capr(view, d1, a.d_cpu, a.d_mem, a.d_gpu) : 0u;
        uint32_t placed = 0;
        int32_t pos = start_e;
        for (; placed < k && pos < ne && pos - start_e < kFifoCache; pos += nt) {
            const int32_t i = pos + tid;
            uint32_t c = 0;
            if (i < ne) c = (i == d1) ? cd1 : a.capr(view, i, 0, 0, 0);
            if (refresh && pos == start_e) {
                bool alive = (i < ne) && !dead_for(gm.exe, view.pair(i), a.use_gpu ? view.gpu(i) : 0, a.use_gpu);
                int32_t f = block_first(sh, buf, alive, i);
                if (tid == 0) sh.first_live_e = f >= 0 ? f : (pos + nt < ne ? pos + nt : ne);
            }
            uint32_t excl, total;
            block_excl_scan(sh, buf, c, excl, total);
            const uint32_t room = k - placed;
            const uint32_t T = total < room ? total : room;
            const uint32_t take = excl >= T ? 0u : ((c < T - excl) ? c : (T - excl));
            if (i - start_e < kFifoCache) cache[i - start_e] = (uint16_t)take;
            if (take != 0) {
                const int32_t node = slot_node[i];
                for (uint32_t t = 0; t < take; ++t) out[placed + excl + t] = node;
            }
            placed += T;
        }
        if (tid == 0) st.nodes += (unsigned long long)((pos < ne ? pos : ne) - start_e);
        if (placed == k) {
            // commit: charge the executors' nodes and the driver's node (sparkpods.go:139-146 / exact)
            bool driver_done = false;
            for (int32_t p0 = start_e; p0 < pos; p0 += nt) {
                const int32_t i = p0 + tid;
                if (i >= ne) continue;
                const uint32_t take = cache[i - start_e];
                if (take != 0) view.charge(i, (FIFO_MODE == 1) ? 1 : (long long)take, a.e_cpu, a.e_mem, a.e_gpu);
                if (i == d1 && (FIFO_MODE == 2 || take == 0)) view.charge(d1, 1, a.d_cpu, a.d_mem, a.d_gpu);
            }
            driver_done = (d1 >= start_e && d1 < pos && d1 < ne);      // its owner thread handled it above
            if (!driver_done && tid == 0) view.charge(d1, 1, a.d_cpu, a.d_mem, a.d_gpu);
            __syncthreads();   // the next application sees the charged snapshot
            return slot_node[d1];
        }
        // executors do not fit with the first fitting driver (or the scan outgrew the cache): decide exactly below
    }

    // ---- phase 1 (see pack_app_impl): P, m1 over a prefix of the executor order, 1024 nodes per step
    unsigned long long P = 0;
    uint32_t m1 = 0;
    int32_t pos = start_e;
    bool early = (k == 0);
    const unsigned long long need = (unsigned long long)k + lmax;
    while (!early && pos < ne) {
        int32_t i = pos + tid;
        uint32_t c = (i < ne) ? a.capr(view, i, 0, 0, 0) : 0u;
        if (cache_ok && i - start_e < kFifoCache) cache[i - start_e] = (uint16_t)c;
        if (pos == start_e) {
            // advance the dead prefix: first position of this step that can still host something
            bool alive = (i < ne) && !dead_for(gm.exe, view.pair(i), a.use_gpu ? view.gpu(i) : 0, a.use_gpu);
            int32_t f = block_first(sh, buf, alive, i);
            if (tid == 0) sh.first_live_e = f >= 0 ? f : (pos + nt < ne ? pos + nt : ne);
        }
        uint32_t sum, cnt;
        if (ALGO == 1) {
            uint32_t excl, total;
            block_excl_scan(sh, buf, c != 0 ? 1u : 0u, excl, total);
            uint32_t r = m1 + excl;
            if (c != 0 && r < k) list[r] = make_int2(i, (int)c);
            cnt = total;
            uint32_t dummy;
            block_reduce2(sh, buf, c, 0u, sum, dummy);
        } else {
            block_reduce2(sh, buf, c, c != 0 ? 1u : 0u, sum, cnt);
        }
        P += sum;
        m1 += cnt;
        pos += nt;
        if (ALGO == 0) early = (P >= need) || (m1 >= k + 1);
        else early = (m1 >= k + 1);
    }
    if (tid == 0) st.nodes += (unsigned long long)((pos < ne ? pos : ne) - start_e);
    const int32_t cached_end = cache_ok ? ((pos - start_e) < kFifoCache ? pos : start_e + kFifoCache) : start_e;
    const bool exact_total = !early;
    if (exact_total && P < k) return -1;

    // ---- phase 2: first feasible driver candidate -------------------------------------------------------
    int32_t dslot = -1;
    for (int32_t j0 = start_d; j0 < g.nd && dslot < 0; j0 += nt) {
        int32_t j = j0 + tid;
        bool feasible = false;
        int32_t ls = -1;
        bool alive = false;
        if (j < g.nd) {
            ls = s.drv_slot[g.dbase + j];
            longlong2 v = view.pair(ls);
            const int64_t gv = a.use_gpu ? view.gpu(ls) : 0;
            alive = !dead_for(gm.drv, v, gv, a.use_gpu);
            feasible = !(a.d_cpu > v.x) && !(a.d_mem > v.y);
            if (a.use_gpu) feasible = feasible && !(a.d_gpu > gv);
            if (feasible && exact_total && ls < ne) {
                uint32_t c0 = a.capr(view, ls, 0, 0, 0);
                uint32_t cdl = a.capr(view, ls, a.d_cpu, a.d_mem, a.d_gpu);
                feasible = (P - c0 + cdl >= k);
            }
        }
        if (j0 == start_d) {
            int32_t f = block_first(sh, buf, alive, j);
            if (tid == 0) sh.first_live_d = f >= 0 ? f : (j0 + nt < g.nd ? j0 + nt : g.nd);
        }
        dslot = block_first(sh, buf, feasible, ls);
        if (tid == 0) st.drivers += (unsigned long long)((g.nd - j0) < nt ? (g.nd - j0) : nt);
    }
    if (dslot < 0) return -1;
    const int32_t driver_node = slot_node[dslot];
    const uint32_t cd = (dslot < ne && k != 0) ? a.capr(view, dslot, a.d_cpu, a.d_mem, a.d_gpu) : 0u;

    // ---- phase 3: emit ExecutorNodes + charge the snapshot -----------------------------------------------
    bool driver_hosts_executor = false;   // per thread; combined below
    if (k != 0) {
        if (ALGO == 0 || early) {
            uint32_t placed = 0;
            for (int32_t p0 = start_e; placed < k && p0 < ne; p0 += nt) {
                int32_t i = p0 + tid;
                uint32_t c = 0;
                if (i == dslot) c = cd;
                else if (i < cached_end) c = cache[i - start_e];
                else if (i < ne) c = a.capr(view, i, 0, 0, 0);
                if (tid == 0 && p0 >= cached_end) st.nodes += (unsigned long long)((ne - p0) < nt ? (ne - p0) : nt);
                const uint32_t unit = (ALGO == 0) ? c : (c != 0 ? 1u : 0u);   // tightly: all it can take; evenly round 1: one
                uint32_t excl, total;
                block_excl_scan(sh, buf, unit, excl, total);
                uint32_t room = k - placed;
                uint32_t T = total < room ? total : room;
                uint32_t take = excl >= T ? 0u : ((unit < T - excl) ? unit : (T - excl));
                if (take != 0) {
                    int32_t node = slot_node[i];
                    for (uint32_t t = 0; t < take; ++t) out[placed + excl + t] = node;
                    if (i == dslot) driver_hosts_executor = true;
                    view.charge(i, (FIFO_MODE == 1) ? 1 : (long long)take, a.e_cpu, a.e_mem, a.e_gpu);
                }
                placed += T;
            }
        } else {
            // general rounds: warp 0 works on the complete candidate list
            __syncthreads();
            if (tid < 32) {
                bool h = evenly_rounds<FIFO_MODE>(list, m1, k, dslot, cd, out, slot_node, lane,
                                                  [&](int32_t local) { view.charge(local, 1, a.e_cpu, a.e_mem, a.e_gpu); });
                driver_hosts_executor = h;
            }
        }
    }
    // ---- charge the driver (sparkpods.go:139-146 / exact) ----------------------------------------------------
    uint32_t hosted, dummy;
    block_reduce2(sh, buf, driver_hosts_executor ? 1u : 0u, 0u, hosted, dummy);   // also orders the executor charges
    if (tid == 0 && (FIFO_MODE == 2 || hosted == 0)) view.charge(dslot, 1, a.d_cpu, a.d_mem, a.d_gpu);
    __syncthreads();   // the next application sees the charged snapshot
    return driver_node;
}

// ---- one application, warp 0 alone ------------------------------------------------------------------------------
// A single warp is bound by the LATENCY of its dependent instruction chain (~650 instructions per application when it
// scans from the batch-wide dead prefix), so the chain is cut where it can be:
//   * the prepared record of the NEXT application is fetched one application ahead -- one coalesced 128-byte load, lane w
//     keeps word w -- and decoded with shuffles: no global-memory latency on the critical path;
//   * availability only ever decreases inside the loop, so "the first driver candidate a driver shape fits on" and "the
//     first node with room for an executor shape" only move forward: warp 0 keeps one cursor per distinct driver /
//     executor request (up to 32 each, one per lane, full tuple compared) and starts both scans there -- typically ONE
//     32-wide step each instead of a walk from the dead prefix;
//   * when everything fits inside the first step the charges are applied straight from registers.
constexpr int kWarpWinE = 32;          // executor steps of 32 nodes the warp tries before it calls the CTA (1 024 nodes)
constexpr int kWarpWinD = 32;          // driver steps of 32 candidates (1 024 candidates)
constexpr int32_t kEscalate = -3;      // "the whole CTA must decide this application" (never stored as a result)

__device__ __forceinline__ void bar_sync_named(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// one cursor per distinct request tuple, entry l lives in lane l
struct ShapeCursors {
    int64_t k0, k1, k2;
    int32_t pos;
    int32_t n;             // entries in use (warp-uniform)
    __device__ __forceinline__ void init() { k0 = k1 = k2 = -1; pos = 0; n = 0; }
    // returns the lane that holds the tuple's cursor (-1: table full) and its value (dflt for a new entry)
    __device__ __forceinline__ int find(int64_t a, int64_t b, int64_t c, int32_t dflt, int32_t& cur, int lane) {
        const unsigned vote = __ballot_sync(kFull, lane < n && k0 == a && k1 == b && k2 == c);
        int src;
        if (vote) src = __ffs(vote) - 1;
        else if (n < kWarp) { src = n; if (lane == src) { k0 = a; k1 = b; k2 = c; pos = dflt; } ++n; }
        else { cur = dflt; return -1; }
        cur = __shfl_sync(kFull, pos, src);
        if (cur < dflt) cur = dflt;      // the batch-wide dead prefix is a lower bound as well
        return src;
    }
};

// the prepared record from the word every lane holds (PrepApp is 32 words)
__device__ __forceinline__ PrepApp decode_prep(uint32_t rec) {
    auto W = [&](int w) { return __shfl_sync(kFull, rec, w); };
    auto W64 = [&](int w) { return (int64_t)(((uint64_t)W(w + 1) << 32) | (uint64_t)W(w)); };
    PrepApp p;
#pragma unroll
    for (int t = 0; t < 3; ++t) {
        p.drv[t] = W64(2 * t);
        p.div[t].magic = (uint64_t)W64(6 + 6 * t);
        p.div[t].e = W64(8 + 6 * t);
        p.div[t].sh = W(10 + 6 * t);
        p.div[t].kind = W(11 + 6 * t);
    }
    p.out_off = W64(24);
    p.count = (int32_t)W(26); p.group = (int32_t)W(27); p.lmax = (int32_t)W(28); p.flags = W(29);
    return p;
}
static_assert(offsetof(PrepApp, div) == 24 && offsetof(PrepApp, out_off) == 96 && offsetof(PrepApp, count) == 104 && offsetof(PrepApp, flags) == 116 &&
              offsetof(DimDiv, e) == 8 && offsetof(DimDiv, sh) == 16 && offsetof(DimDiv, kind) == 20, "decode_prep layout");

// Optimistic single pass, exactly like the first part of fifo_app(): the first driver candidate that FITS is the
// reference's answer whenever the executors fit with it (binpack.go:67-85).  tightly-pack: node n takes min(cap, rest);
// distribute-evenly: one round, every hosting node takes one (distribute_evenly.go:49-70 when k hosting nodes exist).
// Anything else -- no room inside the window budget, executors that do not fit with that driver, several rounds --
// returns kEscalate with NOTHING charged.  Fast arithmetic class only (the general class goes to the CTA).
template <int ALGO, int FIFO_MODE, class V>
__device__ __forceinline__ int32_t fifo_app_warp(const Snapshot& s, const GroupDesc& g, const V& view, const PrepApp& pa,
                                                 int32_t* __restrict__ executor_nodes, uint16_t* __restrict__ cache,
                                                 int32_t start_e, int32_t start_d, ShapeCursors& dcur, ShapeCursors& ecur,
                                                 WarpStats& st, bool drv_identity, int lane) {
    FifoCaps<true> a;
    a.init(&pa, (pa.flags & kAppUsesGpu) || (s.meta->flags & kSnapGpuNegative));
    const uint32_t k = a.k;
    if (k > 0xFFFFu) return kEscalate;                       // takes are cached as uint16
    const int32_t ne = g.ne, nd = g.nd;
    int32_t* out = executor_nodes + pa.out_off;
    const int32_t* slot_node = s.slot_node + g.sbase;
    const bool ug = a.use_gpu;

    // ---- first driver candidate that fits, from this driver shape's cursor -------------------------------------------
    int32_t from_d;
    const int dsrc = dcur.find(a.d_cpu, a.d_mem, a.d_gpu, start_d, from_d, lane);
    int32_t j1 = -1, j0 = from_d;
    for (int w = 0; j0 < nd && j1 < 0 && w < kWarpWinD; ++w, j0 += kWarp) {
        const int32_t j = j0 + lane;
        bool fits = false;
        if (j < nd) {
            const int32_t ls = drv_identity ? j : s.drv_slot[g.dbase + j];
            const longlong2 v = view.pair(ls);
            fits = !(a.d_cpu > v.x) && !(a.d_mem > v.y) && !(ug && a.d_gpu > view.gpu(ls));
        }
        const unsigned vote = __ballot_sync(kFull, fits);
        st.drivers += (unsigned long long)((nd - j0) < kWarp ? (nd - j0) : kWarp);
        if (vote) j1 = j0 + __ffs(vote) - 1;
    }
    if (j1 < 0) {
        if (j0 < nd) return kEscalate;                       // window budget exhausted
        if (lane == dsrc) dcur.pos = nd;                     // this shape fits nowhere any more
        return -1;                                           // no candidate fits at all -> EmptyPackingResult
    }
    if (lane == dsrc) dcur.pos = j1;                         // candidates before j1 can never fit this shape again
    const int32_t d1 = drv_identity ? j1 : s.drv_slot[g.dbase + j1];
    if (k == 0) {                                            // no executors: the driver alone (pack_tightly.go:42-44)
        if (lane == 0) view.charge(d1, 1, a.d_cpu, a.d_mem, a.d_gpu);
        __syncwarp();
        return slot_node[d1];
    }
    const uint32_t cd1 = d1 < ne ? a.capr(view, d1, a.d_cpu, a.d_mem, a.d_gpu) : 0u;

    // ---- executors: 32 nodes per step from this executor shape's cursor -------------------------------------------------
    int32_t from_e;
    const int esrc = ecur.find(a.e_cpu, a.e_mem, a.e_gpu, start_e, from_e, lane);
    uint32_t placed = 0;
    int32_t pos = from_e, first_room = -1;
    for (int w = 0; placed < k && pos < ne && w < kWarpWinE; ++w, pos += kWarp) {
        const int32_t i = pos + lane;
        uint32_t c0 = 0;                                     // capacity without a driver: what the cursor is about
        if (i < ne) c0 = a.capr(view, i, 0, 0, 0);
        const uint32_t c = (i == d1) ? cd1 : c0;
        if (first_room < 0) {
            const unsigned room_vote = __ballot_sync(kFull, c0 != 0);
            if (room_vote) first_room = pos + __ffs(room_vote) - 1;
        }
        const uint32_t unit = (ALGO == 0) ? c : (c != 0 ? 1u : 0u);
        const uint32_t incl = warp_incl_scan(unit, lane);
        const uint32_t total = __shfl_sync(kFull, incl, kWarp - 1);
        const uint32_t room = k - placed;
        const uint32_t T = total < room ? total : room;
        const uint32_t excl = incl - unit;
        const uint32_t take = excl >= T ? 0u : ((unit < T - excl) ? unit : (T - excl));
        if (T != 0) {
            // output j of this step belongs to the first lane whose inclusive prefix exceeds j: shuffle binary search, one
            // coalesced store per 32 outputs (a per-lane loop over `take` serialises up to k stores in one lane)
            const int32_t node = take != 0 ? slot_node[i] : -1;
            for (uint32_t jb = 0; jb < T; jb += kWarp) {
                const uint32_t j = jb + lane;
                int lo = 0;
#pragma unroll
                for (int step = 16; step >= 1; step >>= 1) {
                    const uint32_t v = __shfl_sync(kFull, incl, lo + step - 1);
                    if (v <= j) lo += step;
                }
                const int32_t nd_ = __shfl_sync(kFull, node, lo & 31);
                if (j < T) out[placed + j] = nd_;
            }
        }
        placed += T;
        if (placed == k && w == 0) {
            // the usual case: everything fits inside the first step -> commit straight from registers
            // (sparkpods.go:139-146 / exact accounting)
            st.nodes += (unsigned long long)((pos + kWarp < ne ? pos + kWarp : ne) - from_e);
            if (i < ne) {
                if (take != 0) view.charge(i, (FIFO_MODE == 1) ? 1 : (long long)take, a.e_cpu, a.e_mem, a.e_gpu);
                if (i == d1 && (FIFO_MODE == 2 || take == 0)) view.charge(d1, 1, a.d_cpu, a.d_mem, a.d_gpu);
            }
            const bool in_step = (d1 >= pos && d1 < pos + kWarp && d1 < ne);
            if (!in_step && lane == 0) view.charge(d1, 1, a.d_cpu, a.d_mem, a.d_gpu);
            if (lane == esrc && first_room >= 0) ecur.pos = first_room;      // nodes before it have no room for this shape, for good
            __syncwarp();
            return slot_node[d1];
        }
        cache[pos - from_e + lane] = (uint16_t)take;
    }
    st.nodes += (unsigned long long)((pos < ne ? pos : ne) - from_e);
    if (lane == esrc) ecur.pos = first_room >= 0 ? first_room : (pos < ne ? pos : ne);   // valid whether or not the placement succeeds
    if (placed != k) return kEscalate;                       // nothing has been charged

    // ---- commit after several steps (sparkpods.go:139-146 / exact accounting) ------------------------------------------
    __syncwarp();
    for (int32_t p0 = from_e; p0 < pos; p0 += kWarp) {
        const int32_t i = p0 + lane;
        if (i >= ne) continue;
        const uint32_t take = cache[i - from_e];
        if (take != 0) view.charge(i, (FIFO_MODE == 1) ? 1 : (long long)take, a.e_cpu, a.e_mem, a.e_gpu);
        if (i == d1 && (FIFO_MODE == 2 || take == 0)) view.charge(d1, 1, a.d_cpu, a.d_mem, a.d_gpu);
    }
    const bool driver_done = (d1 >= from_e && d1 < pos && d1 < ne);       // its owner lane handled it above
    if (!driver_done && lane == 0) view.charge(d1, 1, a.d_cpu, a.d_mem, a.d_gpu);
    __syncwarp();                                            // the next application sees the charged snapshot
    return slot_node[d1];
}

// WARP_FIRST = false (GANGPACK_FIFO_WARP=0): warp 0 keeps the queue and the dead prefixes but hands every application to
// the whole CTA -- a second device implementation of the same decision (a template parameter: the default kernel carries
// no extra branch)
template <int ALGO, int FIFO_MODE, bool WARP_FIRST>
__global__ void __launch_bounds__(kFifoThreads, 1) gp_pack_fifo_cta(Snapshot s, const PrepApp* __restrict__ prep,
                                                                    const int32_t* __restrict__ app_group, int32_t n_apps,
                                                                    int32_t* __restrict__ driver_node,
                                                                    int32_t* __restrict__ executor_nodes,
                                                                    int2* __restrict__ scratch,
                                                                    unsigned long long* __restrict__ stats,
                                                                    const GroupMin* __restrict__ gmins,
                                                                    int32_t* __restrict__ app_list, unsigned int* __restrict__ list_cursor) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    FifoScratch& sh = *reinterpret_cast<FifoScratch*>(smem_raw);
    uint16_t* cache = reinterpret_cast<uint16_t*>(smem_raw + 2048);
    longlong2* spair = reinterpret_cast<longlong2*>(smem_raw + 2048 + kFifoCache * sizeof(uint16_t));
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int32_t nt = (int32_t)blockDim.x;
    const int32_t grp = blockIdx.x;
    const GroupDesc g = s.groups[grp];

    // ---- stage the group's executor slots into shared memory (TMA bulk copy) --------------------------
    FifoView view;
    view.sp = spair;
    view.gp = s.pair + g.sbase;
    view.gg = s.gpu + g.sbase;
    view.n_smem = g.ne < kFifoSmemSlots ? g.ne : kFifoSmemSlots;
    view.all_smem = false;
    const uint32_t stage_bytes = (uint32_t)view.n_smem * (uint32_t)sizeof(longlong2);
    if (tid == 0) { mbar_init(&sh.bar, 1); sh.first_live_e = 0; sh.first_live_d = 0; sh.cmd_app = -1; sh.cmd_seq = 0; }
    const GroupMin gm = gmins[grp];
    __syncthreads();
    if (tid == 0 && stage_bytes != 0) {
        mbar_expect_tx(&sh.bar, stage_bytes);
        for (uint32_t off = 0; off < stage_bytes; off += 32768u) {
            uint32_t n = stage_bytes - off < 32768u ? stage_bytes - off : 32768u;
            tma_load_1d(reinterpret_cast<unsigned char*>(spair) + off, reinterpret_cast<const unsigned char*>(view.gp) + off, n, &sh.bar);
        }
    }

    WarpStats st{0, 0};
    int buf = 0;
    // ---- this group's applications in queue order (fitEarlierDrivers walks ONE instance group's queue,
    // sparkpods.go:61): with one group that is every application; otherwise a stable compaction into app_list
    const bool all_mine = (s.n_groups == 1) || app_group == nullptr;     // no group column: every application is in group 0
    int32_t my_cnt = (app_group == nullptr && grp != 0) ? 0 : n_apps;
    const int32_t* mine = nullptr;
    if (!all_mine) {
        int32_t cnt = 0;
        for (int32_t i0 = 0; i0 < n_apps; i0 += nt) {
            const int32_t i = i0 + tid;
            cnt += __syncthreads_count(i < n_apps && app_group[i] == grp);
        }
        if (tid == 0) sh.list_base = (int32_t)atomicAdd(list_cursor, (unsigned int)cnt);
        __syncthreads();
        int32_t* dst = app_list + sh.list_base;
        uint32_t running = 0;
        for (int32_t i0 = 0; i0 < n_apps; i0 += nt) {
            const int32_t i = i0 + tid;
            const bool m = i < n_apps && app_group[i] == grp;
            uint32_t excl, total;
            block_excl_scan(sh, buf, m ? 1u : 0u, excl, total);
            if (m) dst[running + excl] = i;
            running += total;
        }
        my_cnt = cnt;
        mine = dst;
    }
    // driver order == executor order position by position? (the usual case: both come from one sorted list)
    bool ident = true;
    for (int32_t j = tid; j < g.nd; j += nt) ident = ident && (s.drv_slot[g.dbase + j] == j);
    const bool drv_identity = __syncthreads_and(ident) != 0;
    // identical orders and a group that fits the staging area: no slot outside shared memory is ever touched
    view.all_smem = drv_identity && g.nd <= g.ne && g.ne <= kFifoSmemSlots;     // (nd > ne: spare driver-only slots live in global memory)

    if (stage_bytes != 0) mbar_wait(&sh.bar, 0);
    __syncthreads();

    auto run_block = [&](int32_t app, uint32_t seq) -> int32_t {       // every thread of the CTA
        // every helper has read the command word before warp 0 can post the next one, also when fifo_app() leaves
        // without a block-wide barrier of its own (racecheck: cmd_app written while a late helper still read it)
        __syncthreads();
        const PrepApp* pa = prep + app;
        return (pa->flags & kAppFast) ? fifo_app<ALGO, FIFO_MODE, true>(s, g, view, pa, executor_nodes, scratch, cache, sh, buf, st, gm, seq)
                                      : fifo_app<ALGO, FIFO_MODE, false>(s, g, view, pa, executor_nodes, scratch, cache, sh, buf, st, gm, seq);
    };

    if (w == 0) {
        int32_t start_e = 0, start_d = 0;
        bool blocked = false;
        uint32_t seq = 0;
        unsigned long long escalated = 0;
        ShapeCursors dcur, ecur;
        dcur.init(); ecur.init();
        FifoViewS view_s;
        view_s.sp = view.sp; view_s.gg = view.gg;
        // software pipeline: the record of application t+1 (one coalesced 128-byte load, lane w keeps word w) and the index of
        // application t+2 are in flight while application t is decided
        int32_t app = my_cnt > 0 ? (mine ? mine[0] : 0) : 0;
        int32_t app_next = my_cnt > 1 ? (mine ? mine[1] : 1) : 0;
        uint32_t rec = my_cnt > 0 ? reinterpret_cast<const uint32_t*>(prep + app)[lane] : 0u;
        for (int32_t t = 0; t < my_cnt; ++t) {
            const uint32_t rec_next = (t + 1 < my_cnt) ? __ldg(reinterpret_cast<const uint32_t*>(prep + app_next) + lane) : 0u;
            const int32_t app_next2 = (t + 2 < my_cnt) ? (mine ? mine[t + 2] : t + 2) : 0;
            int32_t d;
            if (blocked) d = -2;                                   // never evaluated (resource.go:252)
            else {
                const PrepApp pa = decode_prep(rec);
                const uint32_t fl = pa.flags;
                d = -1;
                if (!(fl & kAppInvalid)) {
                    if ((seq & 15u) == 0) {
                        // every 16th application: advance the dead prefixes -- nodes that can host nothing for ANY application
                        // of the batch (GroupMin); they bound every cursor from below and are where the CTA path starts
                        const bool ug = (fl & kAppUsesGpu) || (s.meta->flags & kSnapGpuNegative);
                        for (int u = 0; u < 8 && start_e < g.ne; ++u) {
                            const int32_t i = start_e + lane;
                            const bool alive = i < g.ne && !dead_for(gm.exe, view.pair(i), ug ? view.gpu(i) : 0, ug);
                            const unsigned vote = __ballot_sync(kFull, alive);
                            if (vote) { start_e += __ffs(vote) - 1; break; }
                            start_e = min(g.ne, start_e + kWarp);
                        }
                        for (int u = 0; u < 8 && start_d < g.nd; ++u) {
                            const int32_t j = start_d + lane;
                            bool alive = false;
                            if (j < g.nd) {
                                const int32_t ls = drv_identity ? j : s.drv_slot[g.dbase + j];
                                alive = !dead_for(gm.drv, view.pair(ls), ug ? view.gpu(ls) : 0, ug);
                            }
                            const unsigned vote = __ballot_sync(kFull, alive);
                            if (vote) { start_d += __ffs(vote) - 1; break; }
                            start_d = min(g.nd, start_d + kWarp);
                        }
                    }
                    int32_t r = kEscalate;                         // general arithmetic class (or !WARP_FIRST): the CTA decides
                    if (WARP_FIRST && (fl & kAppFast))
                        r = view.all_smem ? fifo_app_warp<ALGO, FIFO_MODE>(s, g, view_s, pa, executor_nodes, cache, start_e, start_d, dcur, ecur, st, true, lane)
                                          : fifo_app_warp<ALGO, FIFO_MODE>(s, g, view, pa, executor_nodes, cache, start_e, start_d, dcur, ecur, st, drv_identity, lane);
                    if (r == kEscalate) {
                        ++escalated;
                        if (lane == 0) { sh.first_live_e = start_e; sh.first_live_d = start_d; sh.cmd_app = app; sh.cmd_seq = seq; }
                        __syncwarp();
                        bar_sync_named(1, nt);                     // wake the helper warps
                        r = run_block(app, seq);
                        __syncwarp();
                        start_e = sh.first_live_e; start_d = sh.first_live_d;
                        __syncwarp();                              // every lane has read them before lane 0 writes them again
                    }
                    d = r;
                    ++seq;
                }
                if (d < 0 && !(fl & kAppSkipIfNoFit)) blocked = true;   // resource.go:244-253
            }
            if (lane == 0) driver_node[app] = d;
            app = app_next; app_next = app_next2; rec = rec_next;
        }
        if (lane == 0) { sh.cmd_app = -1; if (escalated) atomicAdd(stats + 2, escalated); }   // stats[2]: applications decided by the whole CTA
        __syncwarp();
        bar_sync_named(1, nt);                                     // release the helpers
    } else {
        for (;;) {
            bar_sync_named(1, nt);
            const int32_t app = sh.cmd_app;
            if (app < 0) break;
            run_block(app, sh.cmd_seq);
        }
    }

    // ---- write the charged slots back (TMA bulk store) ---------------------------------------------------
    __syncthreads();
    if (tid == 0 && stage_bytes != 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (uint32_t off = 0; off < stage_bytes; off += 32768u) {
            uint32_t n = stage_bytes - off < 32768u ? stage_bytes - off : 32768u;
            tma_store_1d(reinterpret_cast<unsigned char*>(view.gp) + off, reinterpret_cast<unsigned char*>(spair) + off, n);
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
    if (tid == 0) {
        atomicAdd(stats + 0, st.nodes);
        atomicAdd(stats + 1, st.drivers);
    }
}

constexpr size_t kFifoSmemBytes = 2048 + kFifoCache * sizeof(uint16_t) + (size_t)kFifoSmemSlots * sizeof(longlong2);

}  // namespace gp

// gangpack_zonefifo.cuh -- the FIFO loop with a single-AZ packer, in ONE launch.
//
// Reference: fitEarlierDrivers (internal/extender/resource.go:224-262) calls binpacker.BinpackFunc once per queued driver;
// with `binpack: single-az-tightly-pack` / `single-az-minimal-fragmentation` that function packs the application in EVERY
// zone and keeps the result with the best average packing efficiency (LIB/binpack/single_az.go:23-55, 75-97), and the
// usage of the winner is subtracted before the next driver is tried (sparkResourceUsage, EXT/sparkpods.go:139-146 +
// SubtractUsageIfExists, LIB/resources/resources.go:129-135).  The zone choice of driver i therefore feeds driver i+1:
// the queue is one sequential chain over the whole cluster (zones are NOT independent queues).
//
// One persistent CTA walks the queue of one instance group (fitEarlierDrivers runs per instance group, resource.go:292-295;
// instance groups share no node, so their CTAs never wait on each other).  CTA b takes ZoneFifoGroup b: its zones, its
// queue and its scratch rows.  Per application:
//   1. warp w packs it in zones w, w + W, ... (snapshot instance group = zone) with the warp-per-application scan of the
//      independent kernels -- here with coherent loads, the availabilities change inside the launch -- into a scratch row
//      per zone; lane 0 of the warp then walks its row for the float64 averages in the reference's operation order;
//   2. __syncthreads; every thread takes the arg-max in zone order (strict '<' against a best that starts at 0.0);
//   3. the winner's warp copies the row out and charges the slots: FIFO_MODE 1 = the reference's map assignment (every
//      DISTINCT executor node once, the driver only when its node hosts no executor), 2 = every pod;
//   4. __syncthreads, next application.  A driver that fits nowhere blocks the queue unless it is young
//      (resource.go:244-253); the applications behind it report -2 like gp_pack_fifo_cta.
//
// az-aware-tightly-pack (ALGO kZoneAzAware, az_aware_pack_tightly.go:27-38) packs the zones with tightly-pack like 1. and,
// when no zone wins in 2., falls back to SparkBinPack(tightlyPackExecutors) over the UNDIVIDED driver / executor orders
// against the availability the loop holds at that point.  Those orders run across the snapshot's groups (zone groups plus
// a trailing group with the nodes no candidate zone contains), so warp 0 scans them through a gather view built once per
// call by gp_build_fallback_view (GatherSlots: position -> slot; CTA b sees the entries of its instance group's orders).
// The fallback's placement lands in row Z and is emitted and charged by the code of 3., so both accounting modes share
// it; it reports zone -1 and zero averages.
#pragma once

#include "gangpack_kernels.cuh"
#include "gangpack_minfrag.cuh"
#include "gangpack_zones.cuh"

namespace gp {

constexpr int kZoneFifoWarps = 16;
constexpr int kZoneFifoThreads = kZoneFifoWarps * 32;
constexpr int kZoneFifoMaxZones = 64;

struct ZoneFifoIn {
    const long long* sched[3];        // SchedulableResources, node-table order (gpu may be NULL = 0)
    const int32_t* node_slot;         // node -> global slot
    int32_t* row_exec;                // per instance group [n_zones (+1 az-aware)][row_pitch] at row_base: ExecutorNodes per zone
    int2* row_list;                   // the same rows: consumed-node list of minimal-fragmentation, NULL for tightly-pack
    const ZoneFifoGroup* groups;      // [gridDim.x]
    const int32_t* queue;             // application indices, instance group after instance group, queue order within each
};

// AvailableResources of a node as the loop currently holds them (the slots are charged inside the launch)
struct SlotAvail {
    const longlong2* pair;
    const int64_t* gpu;
    const int32_t* node_slot;
    __device__ __forceinline__ void load(int32_t n, long long& c, long long& m, long long& g) const {
        const int32_t sl = node_slot[n];
        const longlong2 v = load_pair<true>(pair + sl);
        c = v.x; m = v.y; g = load_gpu<true>(gpu + sl);
    }
};

__device__ __forceinline__ void zone_charge(const Snapshot& s, int32_t slot, long long mult, long long c, long long m, long long g) {
    longlong2 v = load_pair<true>(s.pair + slot);
    v.x -= mult * c; v.y -= mult * m;
    s.pair[slot] = v;
    if (g != 0) s.gpu[slot] = load_gpu<true>(s.gpu + slot) - mult * g;
}

// The fallback view of az-aware-tightly-pack, once per call, one CTA per instance group b, whose undivided orders are
// exec_order[exec_off[b] .. exec_off[b+1]) and drv_order[drv_off[b] .. drv_off[b+1]) (offsets NULL: one instance group,
// the whole orders): fb_exec_slot[i] = node_slot[exec_order[i]], fb_drv_slot[j] = node_slot[drv_order[j]], fb_drv_pos[j]
// = position of drv_order[j] in its instance group's executor order, or -1.  node_pos: [n_nodes] scratch for the node ->
// position scatter; a CTA writes and reads only the entries of its own nodes, and instance groups share no node.
__global__ void __launch_bounds__(1024) gp_build_fallback_view(int32_t n_exec, int32_t n_drv, const int32_t* __restrict__ exec_off,
                                                               const int32_t* __restrict__ drv_off,
                                                               const int32_t* __restrict__ exec_order, const int32_t* __restrict__ drv_order,
                                                               const int32_t* __restrict__ node_slot, int32_t* __restrict__ node_pos,
                                                               int32_t* __restrict__ fb_exec_slot, int32_t* __restrict__ fb_drv_slot,
                                                               int32_t* __restrict__ fb_drv_pos) {
    const int32_t e0 = exec_off ? exec_off[blockIdx.x] : 0, e1 = exec_off ? exec_off[blockIdx.x + 1] : n_exec;
    const int32_t d0 = drv_off ? drv_off[blockIdx.x] : 0, d1 = drv_off ? drv_off[blockIdx.x + 1] : n_drv;
    for (int32_t j = d0 + threadIdx.x; j < d1; j += blockDim.x) node_pos[drv_order[j]] = -1;
    __syncthreads();
    for (int32_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) {
        const int32_t v = exec_order[i];
        node_pos[v] = i - e0;
        fb_exec_slot[i] = node_slot[v];
    }
    __syncthreads();
    for (int32_t j = d0 + threadIdx.x; j < d1; j += blockDim.x) {
        const int32_t v = drv_order[j];
        fb_drv_slot[j] = node_slot[v];
        fb_drv_pos[j] = node_pos[v];
    }
}

// The part of the fallback view `all` that instance group ig's orders cover
__device__ __forceinline__ GatherSlots group_view(const ZoneFifoGroup& ig, const GatherSlots& all) {
    return GatherSlots{all.exec_slot + ig.e0, all.drv_slot + ig.d0, all.drv_pos + ig.d0, ig.ne, ig.nd};
}

// ALGO: 0 tightly-pack, 2 minimal-fragmentation, kZoneAzAware az-aware-tightly-pack.  FIFO_MODE: 1 reference accounting,
// 2 exact.  One CTA per instance group (in.groups).  fb: the fallback view of every instance group, one GatherSlots for
// kZoneAzAware (the row after an instance group's zones is its fallback row), none for the single-AZ packers (so their
// parameter list, and code, stay what they were before the az-aware form existed).
template <int ALGO, int FIFO_MODE, class... FB>
__global__ void __launch_bounds__(kZoneFifoThreads, 1) gp_pack_fifo_zones_cta(Snapshot s, const PrepApp* __restrict__ prep, ZoneFifoIn in,
                                                                              int32_t* __restrict__ zone_out, int32_t* __restrict__ driver_out,
                                                                              int32_t* __restrict__ exec_out, double* __restrict__ avg_out,
                                                                              unsigned long long* __restrict__ stats, FB... fb) {
    constexpr bool kAz = ALGO == kZoneAzAware;
    static_assert(sizeof...(FB) == (kAz ? 1 : 0), "the fallback view goes with az-aware-tightly-pack only");
    __shared__ uint16_t caches[kZoneFifoWarps][kCapCache];
    __shared__ double z_avg[kZoneFifoMaxZones][4];
    __shared__ int32_t z_drv[kZoneFifoMaxZones];
    __shared__ int32_t fb_drv;                        // kAz: driver node of the fallback, -1 = it fits nowhere either
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const ZoneFifoGroup ig = in.groups[blockIdx.x];
    const int32_t Z = ig.n_zones;
    int32_t* const row_exec = in.row_exec + ig.row_base;
    int2* const row_list = in.row_list ? in.row_list + ig.row_base : nullptr;
    GatherSlots view{};
    if constexpr (kAz) view = group_view(ig, fb...);
    const GroupDesc g0 = s.groups[0];
    SlotAvail av;
    av.pair = s.pair; av.gpu = s.gpu; av.node_slot = in.node_slot;
    WarpStats st{0, 0};
    const int snap_flags = s.meta->flags;     // a placement only lands where it fits: no availability turns negative inside the loop
    bool blocked = false;
    for (int32_t qi = ig.q_begin; qi < ig.q_end; ++qi) {
        const int32_t app = in.queue[qi];
        const PrepApp* pa = prep + app;
        const uint32_t fl = pa->flags;
        if (blocked || (fl & kAppInvalid)) {
            if (threadIdx.x == 0) {
                zone_out[app] = -1;
                driver_out[app] = blocked ? -2 : -1;                 // never evaluated (resource.go:252)
                if (avg_out) for (int t = 0; t < 4; ++t) avg_out[4 * (int64_t)app + t] = 0.0;
            }
            continue;
        }
        const int32_t k = pa->count;
        // ---- 1. every zone: pack + averages ---------------------------------------------------------------------------
        for (int32_t z = warp; z < Z; z += kZoneFifoWarps) {
            const int64_t row = (int64_t)z * ig.row_pitch;
            int32_t d;
            if (ALGO == 0 || kAz)
                d = pack_app_impl<0, false, false, false, int32_t, true>(s, pa, row_exec, nullptr, caches[warp], st, lane, snap_flags, g0,
                                                                         ig.zone0 + z, row);
            else
                d = pack_app_minfrag<false, true>(s, pa, row_exec, row_list, st, lane, snap_flags, ig.zone0 + z, row);
            __syncwarp();
            if (lane == 0) {
                z_drv[z] = d;
                if (d >= 0)
                    zone_row_average(av, in.sched, d, row_exec + row, k, pa->drv[0], pa->drv[1], pa->drv[2],
                                     pa->div[0].e, pa->div[1].e, pa->div[2].e, ALGO == 0 || kAz, z_avg[z]);
            }
        }
        __syncthreads();
        // ---- 2. chooseBestResult (single_az.go:75-97), identically in every thread ------------------------------------
        double best = 0.0;
        int32_t best_z = -1;
        for (int32_t z = 0; z < Z; ++z)
            if (z_drv[z] >= 0 && best < z_avg[z][3]) { best = z_avg[z][3]; best_z = z; }
        // ---- 2b. az-aware: no zone won -> warp 0 packs over the undivided orders into row Z (az_aware_pack_tightly.go:33-37)
        int32_t win = best_z;                                        // the row to emit: a zone, or Z for the fallback
        if constexpr (kAz) {
            if (best_z < 0) {
                if (warp == 0) {
                    const int32_t d = pack_app_impl<0, false, false, false, int32_t, true, GatherSlots>(
                        s, pa, row_exec, nullptr, caches[0], st, lane, snap_flags, g0, 0, (int64_t)Z * ig.row_pitch, &view);
                    if (lane == 0) {
                        fb_drv = d;
                        if (stats) atomicAdd(stats + 2, 1ull);   // stats[2]: applications for which the fallback ran
                    }
                }
                __syncthreads();
                if (fb_drv >= 0) win = Z;
            }
        }
        const bool fell_back = kAz && win == Z;
        // ---- 3. the winner's warp emits and charges ---------------------------------------------------------------------
        if (win >= 0 && warp == win % kZoneFifoWarps) {
            const int32_t* ex = row_exec + (int64_t)win * ig.row_pitch;
            int32_t* out = exec_out + pa->out_off;
            const int32_t d = fell_back ? fb_drv : z_drv[win];
            const long long ec = pa->div[0].e, em = pa->div[1].e, eg = pa->div[2].e;
            bool hosts = false;                                      // the driver's node hosts an executor
            for (int32_t t0 = 0; t0 < k; t0 += 32) {
                const int32_t t = t0 + lane;
                if (t < k) {
                    const int32_t n = ex[t];
                    out[t] = n;
                    hosts = hosts || n == d;
                    // one writer per node: the first entry that names it, with the number of entries that do
                    bool first = t == 0 || ex[t - 1] != n;
                    for (int32_t u = 0; first && u + 1 < t; ++u) first = ex[u] != n;
                    if (first) {
                        long long cnt = 1;
                        if (FIFO_MODE == 2) { cnt = 0; for (int32_t u = t; u < k; ++u) cnt += ex[u] == n ? 1 : 0; }
                        zone_charge(s, in.node_slot[n], cnt, ec, em, eg);
                    }
                }
            }
            hosts = __any_sync(kFull, hosts);
            __syncwarp();
            if (lane == 0) {
                if (FIFO_MODE == 2 || !hosts) zone_charge(s, in.node_slot[d], 1, pa->drv[0], pa->drv[1], pa->drv[2]);
                zone_out[app] = fell_back ? -1 : win;
                driver_out[app] = d;
                if (avg_out) for (int t = 0; t < 4; ++t) avg_out[4 * (int64_t)app + t] = fell_back ? 0.0 : z_avg[win][t];
            }
        } else if (win < 0 && threadIdx.x == 0) {
            zone_out[app] = -1;
            driver_out[app] = -1;
            if (avg_out) for (int t = 0; t < 4; ++t) avg_out[4 * (int64_t)app + t] = 0.0;
        }
        if (win < 0 && !(fl & kAppSkipIfNoFit)) blocked = true;       // resource.go:244-253
        __syncthreads();
    }
    if (lane == 0 && stats) { atomicAdd(stats + 0, st.nodes); atomicAdd(stats + 1, st.drivers); }
}

// ---- independent decisions (gp_pack_batch_az_aware) ------------------------------------------------------------------
// Every application is decided against the unmodified snapshot: the zone packs and gp_zone_choose run like
// gp_pack_batch_zones over groups 0..Z-1, then the applications no zone won are listed (in any order: nothing is charged)
// and packed over the undivided orders through the same gather view as the FIFO form.

// listed[0..*n_listed) = the applications with zone[i] == -1; *n_listed starts at 0
__global__ void __launch_bounds__(256) gp_az_fallback_list(int32_t n_apps, const int32_t* __restrict__ zone, int32_t* __restrict__ listed,
                                                            unsigned int* __restrict__ n_listed) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool fb = i < n_apps && zone[i] < 0;
    const unsigned vote = __ballot_sync(kFull, fb);
    if (vote == 0) return;                                     // warp-uniform
    const int lane = threadIdx.x & 31;
    unsigned int base = 0;
    if (lane == 0) base = atomicAdd(n_listed, (unsigned int)__popc(vote));
    base = __shfl_sync(kFull, base, 0);
    if (fb) listed[base + __popc(vote & ((1u << lane) - 1u))] = i;
}

// SparkBinPack(tightlyPackExecutors) over the undivided orders for every listed application: a persistent grid, one warp
// per application claimed from *next.  The driver and ExecutorNodes go straight to the application's own entries of the
// final results (prep[i].out_off is its CSR offset).  MUT = false: nothing writes the slots during the call, so the scan
// takes the read-only loads of the other independent kernels.  stats[2] / [3]: applications / executor-order entries of
// these scans.
constexpr int kAzFallbackThreads = 256;
__global__ void __launch_bounds__(kAzFallbackThreads) gp_pack_az_fallback(Snapshot s, const PrepApp* __restrict__ prep,
                                                                         const int32_t* __restrict__ listed,
                                                                         const unsigned int* __restrict__ n_listed,
                                                                         const __grid_constant__ GatherSlots view,
                                                                         int32_t* __restrict__ drv_node, int32_t* __restrict__ exec_out,
                                                                         unsigned long long* __restrict__ stats,
                                                                         unsigned int* __restrict__ next) {
    __shared__ uint16_t caches[kAzFallbackThreads / 32][kCapCache];
    const unsigned int n = *n_listed;
    if (n == 0) return;
    const int lane = threadIdx.x & 31;
    const int snap_flags = s.meta->flags;
    const GroupDesc none{};                                    // the gather view has no group
    WarpStats st{0, 0};
    unsigned long long apps_done = 0;
    for (;;) {
        unsigned int i = 0;
        if (lane == 0) i = atomicAdd(next, 1u);
        i = __shfl_sync(kFull, i, 0);
        if (i >= n) break;
        const int32_t app = listed[i];
        const PrepApp* pa = prep + app;
        int32_t d = -1;
        if (!(pa->flags & kAppInvalid))
            d = pack_app_impl<0, false, false, false, int32_t, false, GatherSlots>(s, pa, exec_out, nullptr, caches[threadIdx.x >> 5], st,
                                                                                  lane, snap_flags, none, -1, -1, &view);
        if (lane == 0) drv_node[app] = d;
        ++apps_done;
    }
    if (lane == 0) {
        atomicAdd(stats + 0, st.nodes);
        atomicAdd(stats + 1, st.drivers);
        atomicAdd(stats + 2, apps_done);
        atomicAdd(stats + 3, st.nodes);
    }
}

}  // namespace gp

// gangpack_zonelayout.cuh -- the zone-grouped snapshot of the zone-aware packers on the device (gp_prepare_cluster_zones):
// groupNodesByZone over the two priority orders (LIB/binpack/single_az.go:57-73) with the zones in driverZonesInOrder order
// and the zones without executor candidates left out (:36-41), plus, for az-aware-tightly-pack, the trailing group of the
// remaining nodes (az_aware_pack_tightly.go:27-38).
//
//   candidate zones  first[z] = smallest driver-order position of a node of z (atomicMin), has_exec[z] = some executor
//                    candidate lies in z; driver position i is flagged when first[zone] == i && has_exec[zone], and an
//                    exclusive scan of the flags over the driver order numbers the candidate zones in the order of their first
//                    appearance -- O(N) for any number of zones, no sort of the zones.
//   partition        group_rank[node] = the zone's group number, n_zones for the trailing group, -1 for a dropped node; the
//                    label re-sort of gangpack_sort.cuh (a stable re-sort by a per-node rank, -1 last) then partitions each
//                    undivided order, so each group's order is the undivided order restricted to its nodes.
//   offsets          off[g] = number of positions whose rank is below g (binary search: the ranks ascend along the
//                    partitioned order, dropped nodes count as +inf and fall off the end).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace gp {

// ZoneInfo words (device, copied back once at the end of the call)
enum { kZiZones = 0, kZiTrailing = 1, kZiGroups = 2, kZiExec = 3, kZiDrv = 4, kZiWords = 8 };

// first[z] (pre-set to INT_MAX) and has_exec[z] (pre-set to 0) over the two undivided orders; zone == NULL: one zone
__global__ void gp_zone_mark(int32_t n, const int32_t* __restrict__ counts, const int32_t* __restrict__ drv, const int32_t* __restrict__ exe,
                             const int32_t* __restrict__ zone, int32_t* __restrict__ first, uint8_t* __restrict__ has_exec) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (i < counts[0]) atomicMin(first + (zone ? zone[drv[i]] : 0), i);
    if (i < counts[1]) has_exec[zone ? zone[exe[i]] : 0] = 1;
}

// One CTA: exclusive scan of the candidate-zone flags over the driver order.  zone_group[z] (pre-set to -1) = group of a
// candidate zone, zone_of_group[g] (pre-set to -1) = its zone, info[kZiZones] = number of candidate zones.
constexpr int kZoneScanItems = 8;
__global__ void __launch_bounds__(1024) gp_zone_candidates(const int32_t* __restrict__ counts, const int32_t* __restrict__ drv,
                                                           const int32_t* __restrict__ zone, const int32_t* __restrict__ first,
                                                           const uint8_t* __restrict__ has_exec, int32_t* __restrict__ zone_group,
                                                           int32_t* __restrict__ zone_of_group, int32_t* __restrict__ info) {
    __shared__ int32_t wsum[32];
    __shared__ int32_t base;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int32_t n = counts[0];
    if (tid == 0) base = 0;
    __syncthreads();
    for (int32_t p0 = 0; p0 < n; p0 += blockDim.x * kZoneScanItems) {
        const int32_t pb = p0 + tid * kZoneScanItems;
        int32_t z[kZoneScanItems];
        uint32_t f = 0;
#pragma unroll
        for (int t = 0; t < kZoneScanItems; ++t) {
            const int32_t p = pb + t;
            z[t] = 0;
            if (p < n) {
                z[t] = zone ? zone[drv[p]] : 0;
                if (first[z[t]] == p && has_exec[z[t]]) f |= 1u << t;
            }
        }
        const int32_t cnt = __popc(f);
        int32_t inc = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int32_t u = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += u;
        }
        if (lane == 31) wsum[w] = inc;
        __syncthreads();
        int32_t g = base + inc - cnt;
        for (int k = 0; k < w; ++k) g += wsum[k];
#pragma unroll
        for (int t = 0; t < kZoneScanItems; ++t)
            if (f & (1u << t)) { zone_group[z[t]] = g; zone_of_group[g] = z[t]; ++g; }
        __syncthreads();
        if (tid == 0)
            for (int k = 0; k < (int)(blockDim.x >> 5); ++k) base += wsum[k];
        __syncthreads();
    }
    if (tid == 0) info[kZiZones] = base;
}

// group_rank[node] for every node of the two orders: its zone's group, else the trailing group (az_aware) or -1 (dropped).
// info[kZiTrailing] (pre-set to 0) = 1 when some node of either order lies outside every candidate zone.
__global__ void gp_group_rank(int32_t n, const int32_t* __restrict__ counts, const int32_t* __restrict__ drv, const int32_t* __restrict__ exe,
                              const int32_t* __restrict__ zone, const int32_t* __restrict__ zone_group, int32_t az_aware,
                              int32_t* __restrict__ info, int32_t* __restrict__ group_rank) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t rest = az_aware ? info[kZiZones] : -1;
#pragma unroll
    for (int role = 0; role < 2; ++role) {
        if (i >= counts[role]) continue;
        const int32_t v = role == 0 ? drv[i] : exe[i];
        int32_t r = zone_group[zone ? zone[v] : 0];
        if (r < 0) { r = rest; info[kZiTrailing] = 1; }
        group_rank[v] = r;
    }
}

// number of positions of order[0..cnt) whose group is below g (dropped nodes: never)
__device__ __forceinline__ int32_t group_lower_bound(const int32_t* __restrict__ order, int32_t cnt, const int32_t* __restrict__ group_rank,
                                                     int32_t g) {
    int32_t lo = 0, hi = cnt;
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        const int32_t r = group_rank[order[mid]];
        if (r >= 0 && r < g) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// exec_off / drv_off [g_bound + 1] of the partitioned orders: groups past the last one are empty, and off[g_bound] is the
// number of nodes kept.  Thread 0 also derives the number of groups (a single-AZ layout keeps one empty group when no zone
// is a candidate; an az-aware layout has its trailing group when that is non-empty or when no zone is a candidate).
__global__ void gp_group_offsets(int32_t g_bound, const int32_t* __restrict__ counts, const int32_t* __restrict__ drv,
                                 const int32_t* __restrict__ exe, const int32_t* __restrict__ group_rank, int32_t az_aware,
                                 int32_t* __restrict__ exec_off, int32_t* __restrict__ drv_off, int32_t* __restrict__ info) {
    const int32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g > g_bound) return;
    const int32_t d = group_lower_bound(drv, counts[0], group_rank, g), e = group_lower_bound(exe, counts[1], group_rank, g);
    drv_off[g] = d;
    exec_off[g] = e;
    if (g == g_bound) { info[kZiExec] = e; info[kZiDrv] = d; }
    if (g == 0) {
        const int32_t nz = info[kZiZones];
        info[kZiGroups] = az_aware ? nz + ((info[kZiTrailing] || nz == 0) ? 1 : 0) : (nz > 0 ? nz : 1);
    }
}

}  // namespace gp

// gangpack_zonelayout.cuh -- the zone-grouped snapshot of the zone-aware packers on the device (gp_prepare_cluster_zones):
// groupNodesByZone over the two priority orders (LIB/binpack/single_az.go:57-73) with the zones in driverZonesInOrder order
// and the zones without executor candidates left out (:36-41), plus, for az-aware-tightly-pack, the trailing group of the
// remaining nodes (az_aware_pack_tightly.go:27-38).
//
//   candidate zones  first[z] = smallest driver-order position of a node of z (atomicMin), has_exec[z] = some executor
//                    candidate lies in z; driver position i is flagged when first[zone] == i && has_exec[zone], and an
//                    exclusive scan of the flags over the driver order numbers the candidate zones in the order of their first
//                    appearance -- O(N) for any number of zones, no sort of the zones.  With several instance groups z is an
//                    (instance group, zone) pair and a scan over the instance groups places each one's groups after those
//                    of the instance groups before it (gp_zone_candidates).
//   partition        group_rank[node] = the zone's group number, its instance group's trailing group, -1 for a dropped node; the
//                    label re-sort of gangpack_sort.cuh (a stable re-sort by a per-node rank, -1 last) then partitions each
//                    undivided order, so each group's order is the undivided order restricted to its nodes.
//   offsets          off[g] = number of positions whose rank is below g (binary search: the ranks ascend along the
//                    partitioned order, dropped nodes count as +inf and fall off the end).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace gp {

// ZoneInfo words (device, copied back once at the end of the call)
enum { kZiZones = 0, kZiGroups = 2, kZiExec = 3, kZiDrv = 4, kZiWords = 8 };

// Instance groups (gp_prepare_cluster_zones_groups).  Every zone array below is indexed by the (instance group, zone) pair
// p = ig * n_zones + zone (ig NULL: every node in instance group 0; zone NULL: one zone, n_zones 1).  Both undivided orders
// are instance-group-major (the instance group leads the sort key), so a scan along them meets the instance groups in id
// order.  Per instance group g (IgWords, [n_ig + 1] each, pre-zeroed): nz = its candidate zones, trail = some node of its
// orders lies outside them, gbase = its first snapshot group (= group_off), zbase = the candidate zones of the instance
// groups before it, exec_off / drv_off = its range of the undivided orders.
struct IgWords { int32_t *nz, *trail, *gbase, *zbase, *exec_off, *drv_off; };
__device__ __forceinline__ int32_t zone_pair(const int32_t* __restrict__ zone, const int32_t* __restrict__ ig, int32_t n_zones, int32_t v) {
    return (ig ? ig[v] * n_zones : 0) + (zone ? zone[v] : 0);
}
constexpr int32_t kNoFirst = 0x7f7f7f7f;
// gp_prepare_cluster_zones_groups refuses n_ig x (n_zones + 1) above this (n_ig > 1): the pair arrays and the one-CTA
// passes over them are sized by that product
constexpr int64_t kZoneLayoutMaxPairs = (int64_t)1 << 22;              // first[] is filled with 0x7f bytes: no driver candidate in the pair

// first[p] (pre-set to kNoFirst) and has_exec[p] (pre-set to 0) over the two undivided orders
__global__ void gp_zone_mark(int32_t n, const int32_t* __restrict__ counts, const int32_t* __restrict__ drv, const int32_t* __restrict__ exe,
                             const int32_t* __restrict__ zone, const int32_t* __restrict__ ig, int32_t n_zones, int32_t* __restrict__ first,
                             uint8_t* __restrict__ has_exec) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (i < counts[0]) atomicMin(first + zone_pair(zone, ig, n_zones, drv[i]), i);
    if (i < counts[1]) has_exec[zone_pair(zone, ig, n_zones, exe[i])] = 1;
}

// block-wide inclusive scan of one value per thread (blockDim.x a multiple of 32, wsum[32] shared); returns the inclusive
// sum of this thread and leaves the block total in *total of thread 0.  Synchronises.
__device__ __forceinline__ int32_t block_scan(int32_t v, int32_t* wsum, int32_t* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int32_t u = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += u;
    }
    if (lane == 31) wsum[w] = inc;
    __syncthreads();
    for (int k = 0; k < w; ++k) inc += wsum[k];
    if (threadIdx.x == 0) {
        int32_t t = 0;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += wsum[k];
        *total = t;
    }
    __syncthreads();
    return inc;
}

// One CTA.  (1) An exclusive scan of the candidate-zone flags over the driver order numbers the candidate pairs in the
// order of their first appearance: instance group by instance group, and within one in driverZonesInOrder order.
// (2) Per instance group its candidate zones and whether it has a trailing group (a pair with nodes in one order only).
// (3) Scans over the instance groups: each one's groups are its candidate zones, then its extra group -- az_aware: the
// trailing group, present when non-empty or when it has no candidate zone; single-AZ: one empty group when it has no
// candidate zone.  (4) zone_group[p] (pre-set to -1) = the global snapshot group of a candidate pair, zone_of_group[g]
// (pre-set to -1) = its zone.  info[kZiZones] / info[kZiGroups] = the totals.  One instance group needs only (1): the
// numbers are the groups, and gp_group_rank / gp_group_offsets derive the trailing flag and the group count on the way, as
// before instance groups, so that gp_prepare_cluster_zones does no more work than it did.
constexpr int kZoneScanItems = 8;
__global__ void __launch_bounds__(1024) gp_zone_candidates(const int32_t* __restrict__ counts, const int32_t* __restrict__ drv,
                                                           const int32_t* __restrict__ zone, const int32_t* __restrict__ ig,
                                                           int32_t n_zones, int32_t n_ig, int32_t az_aware,
                                                           const int32_t* __restrict__ first, const uint8_t* __restrict__ has_exec,
                                                           int32_t* __restrict__ zone_group, int32_t* __restrict__ zone_of_group,
                                                           IgWords w, int32_t* __restrict__ info) {
    __shared__ int32_t wsum[32];
    __shared__ int32_t base, gbase, zbase;
    const int tid = threadIdx.x;
    const int32_t n = counts[0];
    if (tid == 0) { base = 0; gbase = 0; zbase = 0; }
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
                z[t] = zone_pair(zone, ig, n_zones, drv[p]);
                if (first[z[t]] == p && has_exec[z[t]]) f |= 1u << t;
            }
        }
        const int32_t cnt = __popc(f), b0 = base;          // read before the scan: thread 0 advances base after it
        int32_t total;
        int32_t g = b0 + block_scan(cnt, wsum, &total) - cnt;
#pragma unroll
        for (int t = 0; t < kZoneScanItems; ++t)
            if (f & (1u << t)) {
                if (n_ig == 1) zone_of_group[g] = z[t];    // one instance group: the candidate number is the group
                zone_group[z[t]] = g++;
            }
        if (tid == 0) base += total;
        __syncthreads();
    }
    if (n_ig == 1) {                                     // gbase[0] = zbase[0] = 0 (pre-zeroed); the trailing flag comes
        if (tid == 0) { w.nz[0] = base; info[kZiZones] = base; }   // from gp_group_rank, the group count from gp_group_offsets
        return;
    }
    const int32_t n_pairs = n_ig * n_zones;
    for (int32_t p = tid; p < n_pairs; p += blockDim.x) {
        const int32_t g = p / n_zones;
        const bool d = first[p] != kNoFirst, e = has_exec[p] != 0;
        if (zone_group[p] >= 0) atomicAdd(w.nz + g, 1);
        else if (d || e) w.trail[g] = 1;
    }
    __syncthreads();
    for (int32_t g0 = 0; g0 < n_ig; g0 += blockDim.x) {
        const int32_t g = g0 + tid, gb0 = gbase, zb0 = zbase;
        int32_t nz = 0, grp = 0;
        if (g < n_ig) {
            nz = w.nz[g];
            grp = nz + (az_aware ? ((w.trail[g] || nz == 0) ? 1 : 0) : (nz == 0 ? 1 : 0));
        }
        int32_t tg, tz;
        const int32_t ginc = block_scan(grp, wsum, &tg), zinc = block_scan(nz, wsum, &tz);
        if (g < n_ig) { w.gbase[g] = gb0 + ginc - grp; w.zbase[g] = zb0 + zinc - nz; }
        if (tid == 0) { gbase += tg; zbase += tz; }
        __syncthreads();
    }
    for (int32_t p = tid; p < n_pairs; p += blockDim.x) {
        const int32_t c = zone_group[p];
        if (c < 0) continue;
        const int32_t g = p / n_zones;
        const int32_t grp = c - w.zbase[g] + w.gbase[g];
        zone_group[p] = grp;
        zone_of_group[grp] = p - g * n_zones;
    }
    if (tid == 0) {
        w.gbase[n_ig] = gbase;
        info[kZiZones] = base;
        info[kZiGroups] = gbase;
    }
}

// group_rank[node] for every node of the two orders: its pair's group, else its instance group's trailing group (az_aware)
// or -1 (dropped), and w.trail of that instance group.  The ranks ascend with the instance group.
__global__ void gp_group_rank(int32_t n, const int32_t* __restrict__ counts, const int32_t* __restrict__ drv, const int32_t* __restrict__ exe,
                              const int32_t* __restrict__ zone, const int32_t* __restrict__ ig, int32_t n_zones,
                              const int32_t* __restrict__ zone_group, int32_t az_aware, IgWords w, int32_t* __restrict__ group_rank) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
#pragma unroll
    for (int role = 0; role < 2; ++role) {
        if (i >= counts[role]) continue;
        const int32_t v = role == 0 ? drv[i] : exe[i];
        int32_t r = zone_group[zone_pair(zone, ig, n_zones, v)];
        if (r < 0) {
            const int32_t g = ig ? ig[v] : 0;
            r = az_aware ? w.gbase[g] + w.nz[g] : -1;
            w.trail[g] = 1;                              // (already set by gp_zone_candidates with several instance groups)
        }
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
// number of positions of an undivided order whose instance group is below g (ig NULL: one instance group)
__device__ __forceinline__ int32_t ig_lower_bound(const int32_t* __restrict__ order, int32_t cnt, const int32_t* __restrict__ ig, int32_t g) {
    if (!ig) return g == 0 ? 0 : cnt;
    int32_t lo = 0, hi = cnt;
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (ig[order[mid]] < g) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// exec_off / drv_off [g_bound + 1] of the partitioned orders: groups past the last one are empty, and off[g_bound] is the
// number of nodes kept (info[kZiExec] / info[kZiDrv]).  Threads g <= n_ig (<= g_bound) also write the instance groups'
// ranges of the undivided orders udrv / uexe.  One instance group: thread 0 also derives the number of groups (a single-AZ
// layout keeps one empty group when no zone is a candidate; an az-aware layout has its trailing group when that is
// non-empty or when no zone is a candidate).
__global__ void gp_group_offsets(int32_t g_bound, const int32_t* __restrict__ counts, const int32_t* __restrict__ drv,
                                 const int32_t* __restrict__ exe, const int32_t* __restrict__ group_rank, int32_t az_aware,
                                 int32_t* __restrict__ exec_off, int32_t* __restrict__ drv_off, int32_t* __restrict__ info, int32_t n_ig,
                                 const int32_t* __restrict__ ig, const int32_t* __restrict__ udrv, const int32_t* __restrict__ uexe,
                                 IgWords w) {
    const int32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g > g_bound) return;
    const int32_t d = group_lower_bound(drv, counts[0], group_rank, g), e = group_lower_bound(exe, counts[1], group_rank, g);
    drv_off[g] = d;
    exec_off[g] = e;
    if (g == g_bound) { info[kZiExec] = e; info[kZiDrv] = d; }
    if (g == 0 && n_ig == 1) {
        const int32_t nz = info[kZiZones];
        const int32_t groups = az_aware ? nz + ((w.trail[0] || nz == 0) ? 1 : 0) : (nz > 0 ? nz : 1);
        info[kZiGroups] = groups;
        w.gbase[1] = groups;
    }
    if (g <= n_ig) {
        w.drv_off[g] = ig_lower_bound(udrv, counts[0], ig, g);
        w.exec_off[g] = ig_lower_bound(uexe, counts[1], ig, g);
    }
}

}  // namespace gp

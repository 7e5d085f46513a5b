// gangpack_reconcile.cuh -- the failover reconciler's node choice for stale drivers on the device.
//
// Reference (EXT = internal/extender, LIB = vendor/github.com/palantir/k8s-spark-scheduler-lib/pkg):
//   syncResourceReservationsAndDemands    EXT/failover.go:43-82
//   syncResourceReservations              EXT/failover.go:118-160  (available[g].Sub(reserved) at :159)
//   availableResourcesPerInstanceGroup    EXT/failover.go:286-323
//   constructResourceReservation          EXT/failover.go:348-390
//   findNodes                             EXT/failover.go:409-436
//
// Node order: schedulable, ready nodes by ascending (instance group, creation descending, node-table index) -- the
// newest-first sort.Slice of :292-294 followed by the order-keeping partition of :312-313 (DESIGN §2.3 argues the tie order).
// findNodes in closed form (DESIGN §2.3): with c(n) = cap(n|0) against the group's current availability and rem the executors
// still to place when the walk reaches n, node n takes t = min(c(n), rem) executors and is charged (t + 1) x exe when t < rem
// (the addition that failed stays in `reserved`), t x exe when t == rem (the walk returned); later nodes are untouched.
//
// Kernels (one stream, no host round trip between them):
//   gp_rc_node_keys    thread per node: key (group, -creation, index); unschedulable / not-ready nodes get group n_groups
//   gp_sort_tiles / gp_rank_by_search / gp_scatter_order over those keys: the per-group orders, back to back
//   gp_rc_app_list     identity list of the stale drivers; gp_label_keys .. gp_label_scatter partition it stably by group
//   gp_rc_offsets      thread per group: node and driver offsets by binary search (group_lower_bound)
//   gp_rc_loop         persistent: one CTA claims one instance group at a time and runs its drivers in call order
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "gangpack_kernels.cuh"
#include "gangpack_minfrag.cuh"
#include "gangpack_resched.cuh"
#include "gangpack_sort.cuh"
#include "gangpack_zonelayout.cuh"

namespace gp {

constexpr int kRcThreads = 256;

enum : int { kRcErrDomain = 1 };        // an availability the loop read or wrote lies outside the exact-int64 domain

struct ReconKey {          // 16 bytes; (group, index) is unique
    long long creation;
    uint32_t group;        // n_groups: dropped (unschedulable or not ready)
    int32_t idx;
};
__device__ __forceinline__ bool key_less(const ReconKey& a, const ReconKey& b) {
    if (a.group != b.group) return a.group < b.group;
    if (a.creation != b.creation) return a.creation > b.creation;      // newest first
    return a.idx < b.idx;
}
__device__ __forceinline__ ReconKey key_max(const ReconKey*) {
    ReconKey k; k.creation = -0x7fffffffffffffffLL - 1; k.group = 0xffffffffu; k.idx = 0x7fffffff; return k;
}

// grp[i] = the node's group, or n_groups when it is unschedulable or not ready (sorted last, in no group's range)
__global__ void gp_rc_node_keys(int32_t n, int32_t n_groups, const int32_t* __restrict__ node_group, const long long* __restrict__ creation,
                                const uint8_t* __restrict__ unschedulable, const uint8_t* __restrict__ ready,
                                ReconKey* __restrict__ keys, int32_t* __restrict__ grp) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool keep = !(unschedulable && unschedulable[i]) && (ready ? ready[i] != 0 : true);
    const int32_t g = keep ? node_group[i] : n_groups;
    ReconKey k; k.creation = creation[i]; k.group = (uint32_t)g; k.idx = i;
    keys[i] = k;
    grp[i] = g;
}

__global__ void gp_rc_app_list(int32_t q, int32_t* __restrict__ list, int32_t* __restrict__ count) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < q) list[i] = i;
    if (i == 0) *count = q;
}

// noff / aoff [n_groups + 1]: group g owns order[noff[g]..noff[g+1]) and apps[aoff[g]..aoff[g+1])
__global__ void gp_rc_offsets(int32_t n_groups, int32_t n, const int32_t* __restrict__ order, const int32_t* __restrict__ node_grp,
                              int32_t q, const int32_t* __restrict__ apps, const int32_t* __restrict__ app_grp,
                              int32_t* __restrict__ noff, int32_t* __restrict__ aoff) {
    const int32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g > n_groups) return;
    noff[g] = group_lower_bound(order, n, node_grp, g);
    aoff[g] = q ? group_lower_bound(apps, q, app_grp, g) : 0;
}

struct RcLoopIn {
    long long* avail;              // [3][n] availability, charged in place
    const int32_t* order;          // [n] per-group node orders, back to back
    const int32_t* noff;           // [n_groups + 1]
    const int32_t* apps;           // [q] stale drivers grouped by instance group, call order inside a group
    const int32_t* aoff;           // [n_groups + 1]
    const long long* exe;          // [3][q] executor requests
    const int32_t* count;          // [q] executors to place
    const long long* out_off;      // [q] first ExecutorNodes entry of each driver
    int32_t* placed;               // [q]
    int32_t* exec_nodes;           // [sum count]
    unsigned int* claim;           // group claim counter
    int* err;
    int32_t n, q, n_groups;
};

// findNodes for every stale driver of a group, one group per CTA at a time.  Per driver the CTA walks the group's order in
// tiles of kRcThreads nodes: each thread takes m = min(c(n), rem at the tile) for its node, a block scan with the tile's carry
// finds how many executors the walk still owes when it reaches each node, the completing node is the first whose inclusive
// sum reaches that, and every node the walk reaches -- zero-capacity ones included -- is charged by its own thread.  No node
// may be skipped: a node with no room is still charged one executor.  Availability is read with plain (coherent) loads: this
// CTA is its only writer.
__global__ void __launch_bounds__(kRcThreads) gp_rc_loop(RcLoopIn in) {
    __shared__ unsigned long long s_incl[kRcThreads];
    __shared__ unsigned long long s_wsum[kRcThreads / kWarp];
    __shared__ int32_t s_node[kRcThreads];
    __shared__ int32_t s_g;
    const int tid = threadIdx.x, lane = tid & (kWarp - 1), w = tid / kWarp;
    const size_t N = (size_t)in.n, Q = (size_t)in.q;
    for (;;) {
        if (tid == 0) s_g = (int32_t)atomicAdd(in.claim, 1u);
        __syncthreads();
        const int32_t g = s_g;
        if (g >= in.n_groups) return;
        const int32_t n0 = in.noff[g], n1 = in.noff[g + 1];
        for (int32_t a = in.aoff[g]; a < in.aoff[g + 1]; ++a) {
            const int32_t i = in.apps[a];
            const int32_t k = in.count[i];
            if (n0 == n1 || k == 0) {                 // no schedulable, ready node: "instance group not found" (:358-362)
                if (tid == 0) in.placed[i] = n0 == n1 ? -1 : 0;
                continue;
            }
            long long e[3];
            DimDiv dv[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) { e[d] = in.exe[d * Q + i]; dv[d] = make_dimdiv(e[d]); }
            const long long off = in.out_off[i];
            unsigned long long done = 0;              // executors placed before the current tile (uniform)
            for (int32_t p0 = n0; p0 < n1; p0 += kRcThreads) {
                const int32_t p = p0 + tid;
                const bool has = p < n1;
                const int32_t v = has ? in.order[p] : -1;
                const unsigned long long rem0 = (unsigned long long)k - done;
                long long av[3] = {0, 0, 0};
                unsigned long long m = 0;
                if (has) {
                    uint64_t c = kCapInf;
#pragma unroll
                    for (int d = 0; d < 3; ++d) { av[d] = in.avail[d * N + v]; c = min(c, cap_dim_u(av[d], dv[d])); }
                    m = min((unsigned long long)c, rem0);
                }
                // block inclusive scan of m (at most kRcThreads x 2^24: 64-bit)
                unsigned long long incl = m;
#pragma unroll
                for (int d = 1; d < kWarp; d <<= 1) {
                    const unsigned long long t = __shfl_up_sync(kFull, incl, d);
                    if (lane >= d) incl += t;
                }
                if (lane == kWarp - 1) s_wsum[w] = incl;
                __syncthreads();
                unsigned long long total = 0;
#pragma unroll
                for (int k2 = 0; k2 < kRcThreads / kWarp; ++k2) {
                    const unsigned long long s = s_wsum[k2];
                    if (k2 < w) incl += s;
                    total += s;
                }
                const unsigned long long excl = incl - m;
                if (has && excl < rem0) {             // the walk reaches this node
                    const unsigned long long rem = rem0 - excl;
                    const unsigned long long t = min(m, rem);
                    const long long charge = (long long)(t < rem ? t + 1 : t);
                    bool bad = false;
#pragma unroll
                    for (int d = 0; d < 3; ++d) {
                        // t x e <= a when a >= 0 and t = 0 when a < 0: the product stays below 2^62, the difference above -2^62
                        const long long nv = av[d] - charge * e[d];
                        bad |= av[d] >= kMaxQuantity || av[d] <= -kMaxQuantity || nv <= -kMaxQuantity;
                        if (e[d] != 0) in.avail[d * N + v] = nv;
                    }
                    if (bad) atomicOr(in.err, kRcErrDomain);
                }
                s_incl[tid] = min(incl, rem0);
                s_node[tid] = v;
                __syncthreads();
                // ExecutorNodes of the tile, node-major: entry j belongs to the first node whose inclusive sum exceeds j
                const unsigned long long tile_placed = min(total, rem0);
                for (unsigned long long j = tid; j < tile_placed; j += kRcThreads) {
                    int lo = 0, hi = kRcThreads - 1;
                    while (lo < hi) {
                        const int mid = (lo + hi) >> 1;
                        if (s_incl[mid] > j) hi = mid; else lo = mid + 1;
                    }
                    in.exec_nodes[off + (long long)(done + j)] = s_node[lo];
                }
                done += tile_placed;
                __syncthreads();                      // s_incl / s_node / s_wsum and the charges are complete for the next step
                if (done == (unsigned long long)k) break;
            }
            if (tid == 0) in.placed[i] = (int32_t)done;
        }
        __syncthreads();                              // s_g is rewritten by the next claim
    }
}

}  // namespace gp

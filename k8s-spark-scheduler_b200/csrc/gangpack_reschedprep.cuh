// gangpack_reschedprep.cuh -- rescheduleExecutor (SURVEY §8f row f4) straight from the reservations: the executor Predicate
// without a usable reservation, from the node table to the node choice, without sorting the nodes.
//
// Reference (all under /root/reference; EXT = internal/extender, LIB = vendor/github.com/palantir/k8s-spark-scheduler-lib/pkg):
//   rescheduleExecutor                                   EXT/resource.go:594-673
//   filterNodesToZone                                    EXT/resource.go:463-478
//   rescheduleExecutorWithMinimalFragmentation           EXT/resource.go:675-705
//   PotentialNodes / scheduleContextLessThan             internal/sort/nodesorting.go:41-64, 83-93, 161-200
//
// The reference sorts every node (PotentialNodes) and then takes ONE decision over that order.  A decision needs no order:
// with K(n) = (L, P, mem, cpu, name rank) -- L the executor label key (unknown last; 0 when no label is configured), P the
// zone priority, mem / cpu the metadata availability -- K is unique (name ranks are) and the executor order is ascending K
// (a stable re-sort by label rank of an order sorted by (P, mem, cpu, name) is a sort by (L, P, mem, cpu, name)).  So
//   first fit:              the candidate with the smallest K among those the executor fits on (:657-662);
//   minimal fragmentation:  the smallest (not hosting, capacity, K) among the candidates with capacity >= 1 (:688-699 is a
//                           running lexicographic minimum over the order, DESIGN.md §2).
// Kernels: member mask + zone totals over the kept nodes, the zone priority (gp_zone_priority), one 64-byte record per
// node, and one CTA per executor that arg-mins over the records (a CTA rather than a warp: one executor over 50 000 nodes
// is 196 records per thread instead of 1 563).
//
// Ambiguity (SURVEY App. B6): scheduleContextLessThan leaves two nodes unordered when their zone priority, memory and cpu
// agree but their gpu does not, and sort.Slice is unstable.  The decision is then the reference's own unspecified choice
// iff another node that qualifies equally well -- same (class, capacity) for minimal fragmentation -- sits in the winner's
// group (same L, P, mem, cpu) with a different gpu.  The arg-min carries that flag as part of its monoid: merging two
// partial winners of one group sets it when either had it or their gpus differ.
#pragma once

#include "gangpack_resched.cuh"
#include "gangpack_sort.cuh"

namespace gp {

struct RpNode {            // 64 bytes, one per node of the caller's table
    long long mem, cpu;    // metadata availability: alloc - (reservations + overhead)   (key)
    long long gpu;         // metadata availability gpu (ambiguity only)
    long long v[3];        // first fit: availableResources (overhead counted twice on reserved nodes, App. B7);
                           // minimal fragmentation: metadata availability - overhead (GetNodeCapacities' "reserved", :682)
    uint32_t L;            // executor label key: rank, unknown = 0x7fffffff (createLabelLessThanFunction); 0 = no label
    int32_t P;             // zone priority
    int32_t nr;            // name rank
    int32_t cand;          // kept by the scope, schedulable and ready (PotentialNodes' executor candidates, :55-57)
};
static_assert(sizeof(RpNode) == 64, "one record = two 32-byte sectors");

__device__ __forceinline__ bool rp_member(int32_t i, int32_t keep, const int32_t* __restrict__ tz) {
    return keep < 0 || tz[i] == keep;
}

// getAvailableResourcesByAZ (nodesorting.go:124-134) over the nodes filterNodesToZone keeps
__global__ void gp_rp_zone_totals(int32_t n, const long long* __restrict__ cpu, const long long* __restrict__ mem,
                                  const int32_t* __restrict__ zone, int32_t keep, const int32_t* __restrict__ tz,
                                  unsigned long long* __restrict__ tot /* [kZoneTotWords * Z] */) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !rp_member(i, keep, tz)) return;
    zone_total_add(tot, zone[i], mem[i], cpu[i]);
}

struct RpNodeIn {
    const long long* avail;          // [3][n] metadata availability
    const long long* ff;             // [3][n] first-fit availability, or null (minimal fragmentation)
    const long long* over[3];        // overhead per dimension, or null (= 0); minimal fragmentation only
    const int32_t* zone;             // or null (one zone)
    const int32_t* prio;             // [n_zones]
    const int32_t* name_rank;        // or null (index order)
    const uint8_t* unschedulable;    // or null
    const uint8_t* ready;            // or null
    const int32_t* label_rank;       // or null
    const int32_t* tz;               // topology zone per node (scope), read when keep >= 0
    int32_t keep;
    int32_t n;
    int* err;                        // kFeErr* bits of the availability stage
};

__global__ void gp_rp_nodes(RpNodeIn in, RpNode* __restrict__ out) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= in.n) return;
    const size_t N = (size_t)in.n;
    RpNode r;
    r.mem = in.avail[N + i]; r.cpu = in.avail[i]; r.gpu = in.avail[2 * N + i];
#pragma unroll
    for (int d = 0; d < 3; ++d)
        r.v[d] = in.ff ? in.ff[(size_t)d * N + i] : in.avail[(size_t)d * N + i] - (in.over[d] ? in.over[d][i] : 0);
    // availability and overhead are inside the domain (or *err is set already), so the difference did not wrap
    if (!in_domain(r.v[0]) || !in_domain(r.v[1]) || !in_domain(r.v[2])) atomicOr(in.err, kFeErrResult);
    const int32_t lr = in.label_rank ? in.label_rank[i] : 0;
    r.L = lr < 0 ? 0x7fffffffu : (uint32_t)lr;
    r.P = in.zone ? in.prio[in.zone[i]] : 0;
    r.nr = in.name_rank ? in.name_rank[i] : i;
    r.cand = rp_member(i, in.keep, in.tz) && !(in.unschedulable && in.unschedulable[i]) && (in.ready ? in.ready[i] != 0 : true);
    out[i] = r;
}

// A partial winner: the smallest (cap, L, P, mem, cpu, nr) seen, and whether its group (cap, L, P, mem, cpu) holds a
// qualifying node with another gpu.  idx < 0: nothing seen.
struct RpBest {
    unsigned long long cap;
    long long mem, cpu, gpu;
    uint32_t L;
    int32_t P, nr, idx, amb;
};

__device__ __forceinline__ void rp_none(RpBest& b) { b.cap = 0; b.mem = b.cpu = b.gpu = 0; b.L = 0; b.P = 0; b.nr = 0; b.idx = -1; b.amb = 0; }

// 1: group(a) < group(b), -1: group(b) < group(a), 0: same group
__device__ __forceinline__ int rp_group_cmp(const RpBest& a, const RpBest& b) {
    if (a.cap != b.cap) return a.cap < b.cap ? 1 : -1;
    if (a.L != b.L) return a.L < b.L ? 1 : -1;
    if (a.P != b.P) return a.P < b.P ? 1 : -1;
    if (a.mem != b.mem) return a.mem < b.mem ? 1 : -1;
    if (a.cpu != b.cpu) return a.cpu < b.cpu ? 1 : -1;
    return 0;
}

__device__ __forceinline__ void rp_merge(RpBest& a, const RpBest& b) {
    if (b.idx < 0) return;
    if (a.idx < 0) { a = b; return; }
    const int g = rp_group_cmp(a, b);
    if (g < 0) { a = b; return; }
    if (g > 0) return;
    const int32_t amb = a.amb | b.amb | (a.gpu != b.gpu ? 1 : 0);
    if (b.nr < a.nr) a = b;
    a.amb = amb;
}

__device__ __forceinline__ RpBest rp_shfl(const RpBest& v, int d) {
    RpBest o;
    o.cap = __shfl_xor_sync(kFull, v.cap, d);
    o.mem = __shfl_xor_sync(kFull, v.mem, d);
    o.cpu = __shfl_xor_sync(kFull, v.cpu, d);
    o.gpu = __shfl_xor_sync(kFull, v.gpu, d);
    o.L = __shfl_xor_sync(kFull, v.L, d);
    o.P = __shfl_xor_sync(kFull, v.P, d);
    o.nr = __shfl_xor_sync(kFull, v.nr, d);
    o.idx = __shfl_xor_sync(kFull, v.idx, d);
    o.amb = __shfl_xor_sync(kFull, v.amb, d);
    return o;
}

constexpr int kRpThreads = 256;

// CTA-wide reduction; every thread returns the CTA's winner.  `sm` holds one partial per warp.
__device__ __forceinline__ RpBest rp_block_min(RpBest b, RpBest* sm) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) rp_merge(b, rp_shfl(b, d));
    if (lane == 0) sm[w] = b;
    __syncthreads();
    RpBest r = sm[0];
    for (int k = 1; k < kRpThreads / 32; ++k) rp_merge(r, sm[k]);
    __syncthreads();                    // sm is reused by the next reduction
    return r;
}

struct RpDecideIn {
    const int64_t* exe;              // [3][q]
    const int64_t* host_off;         // [q+1] or null
    const int32_t* host_nodes;       // caller node indices
    int32_t n, q;
};

// One CTA per executor (grid-stride): the arg-min of DESIGN.md §2 over the node records.
template <bool MINFRAG>
__global__ void __launch_bounds__(kRpThreads) gp_rp_decide(const RpNode* __restrict__ rec, RpDecideIn in, int32_t* __restrict__ node_out,
                                                           uint8_t* __restrict__ amb_out) {
    __shared__ RpBest sm[kRpThreads / 32];
    const size_t Q = (size_t)in.q;
    for (int32_t x = blockIdx.x; x < in.q; x += gridDim.x) {
        const int64_t ec = in.exe[x], em = in.exe[Q + x], eg = in.exe[2 * Q + x];
        DimDiv dv[3];
        if (MINFRAG) { dv[0] = make_dimdiv(ec); dv[1] = make_dimdiv(em); dv[2] = make_dimdiv(eg); }
        // qualifies: first fit = fits (!GreaterThan, resources.go:239-241); minimal fragmentation = capacity >= 1 (:687)
        auto visit = [&](int32_t i, RpBest& b) {
            const RpNode r = rec[i];
            if (!r.cand) return;
            unsigned long long c = 0;
            if (MINFRAG) {
                c = min(min(cap_dim_u(r.v[0], dv[0]), cap_dim_u(r.v[1], dv[1])), cap_dim_u(r.v[2], dv[2]));
                if (c < 1) return;
            } else if (ec > r.v[0] || em > r.v[1] || eg > r.v[2]) {
                return;
            }
            RpBest o;
            o.cap = c; o.mem = r.mem; o.cpu = r.cpu; o.gpu = r.gpu; o.L = r.L; o.P = r.P; o.nr = r.nr; o.idx = i; o.amb = 0;
            rp_merge(b, o);
        };
        RpBest best;
        rp_none(best);
        if (MINFRAG && in.host_off) {
            // class 0 first: a hosting node with capacity >= 1 beats every other node (:693-695)
            for (int64_t t = in.host_off[x] + threadIdx.x; t < in.host_off[x + 1]; t += blockDim.x) visit(in.host_nodes[t], best);
            best = rp_block_min(best, sm);
        }
        if (best.idx < 0) {             // no hosting node qualifies: every qualifying node is of class 1
            for (int32_t i = threadIdx.x; i < in.n; i += blockDim.x) visit(i, best);
            best = rp_block_min(best, sm);
        }
        if (threadIdx.x == 0) {
            node_out[x] = best.idx;
            if (amb_out) amb_out[x] = best.idx >= 0 && best.amb ? 1 : 0;
        }
    }
}

}  // namespace gp

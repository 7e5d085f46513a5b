// gangpack_sort.cuh -- SURVEY §8f row f1: NodeSorter.PotentialNodes (internal/sort/nodesorting.go:41-122,
// 161-200) on the device -- the step immediately before the packing hot path.
//
//   node priority order = ascending (AZ priority, available memory, available CPU, node name)      :83-93
//   AZ priority         = rank of the zone by (sum of available memory, sum of available CPU)       :102-115
//   driver candidates   = that order restricted to kube-scheduler's NodeNames                        :52-54
//   executor candidates = that order restricted to schedulable && ready nodes                        :55-57
//   optional stable re-sort of either list by the rank of a configured label value                  :61-62, 161-200
//
// The key is a strict total order (node names are unique), so the position of a node is the number of nodes with a
// smaller key.  Two kernels: (1) every CTA sorts one tile of 4 096 keys in shared memory (bitonic network, 96 KB);
// (2) every node binary-searches its key in every sorted tile and adds up the lower bounds -- N x (N / 4096) x 12
// dependent steps instead of the N^2 comparisons of an enumeration sort (10 000 nodes: 3 tiles; 50 000: 13; 500 000:
// 123), no atomics, no multi-pass data movement, deterministic.  The same primitive re-sorts a candidate list stably
// by label rank (key = (rank, position)).
//
// Where the reference's comparator leaves the order undefined (equal (memory, cpu) but different gpu:
// scheduleContextLessThan is not a strict weak order there, SURVEY App. B6; equal zone totals) this
// implementation orders by node name / by zone id -- and REPORTS it (gp_sort_input.undefined_ties) so that the shim can
// route such a Predicate to the Go sorter if it wants the reference's (unspecified) choice.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "gangpack_kernels.cuh"
#include "gangpack_tilesort.cuh"

namespace gp {

// ---- exact sums of signed 64-bit terms ------------------------------------------------------------------------------
// The reference adds resource.Quantity values, which have no bound; a 64-bit atomicAdd wraps.  As in gangpack_overhead.cuh a
// sum is kept in two words, each with an atomicAdd of its own: `lo` sums the terms' low 32 bits, `hi` their (arithmetic) high
// halves.  With fewer than 2^31 terms lo < 2^63 and |hi| < 2^62 for ANY int64 terms, so neither word wraps, and
// sum = hi * 2^32 + lo exactly.
__device__ __forceinline__ void exact_add(unsigned long long* lo, unsigned long long* hi, long long v) {
    const unsigned long long l = (unsigned long long)v & 0xffffffffull;
    const long long h = v >> 32;
    if (l) atomicAdd(lo, l);
    if (h) atomicAdd(hi, (unsigned long long)h);
}
struct ExactSum {          // hi * 2^32 + lo, normalised: comparing (hi, lo) compares the sums
    long long hi;
    uint32_t lo;
};
__device__ __forceinline__ ExactSum exact_sum(unsigned long long lo, unsigned long long hi) {
    ExactSum s; s.hi = (long long)hi + (long long)(lo >> 32); s.lo = (uint32_t)lo;
    return s;
}
__device__ __forceinline__ int exact_cmp(const ExactSum& a, const ExactSum& b) {
    return a.hi != b.hi ? (a.hi < b.hi ? -1 : 1) : (a.lo != b.lo ? (a.lo < b.lo ? -1 : 1) : 0);
}
__device__ __forceinline__ bool in_domain(long long v) { return v > -kMaxQuantity && v < kMaxQuantity; }
// *v = the sum when it lies inside the exact-int64 domain (|sum| < 2^61)
__device__ __forceinline__ bool exact_value(const ExactSum& s, long long* v) {
    constexpr long long lim = kMaxQuantity >> 32;
    if (s.hi < -lim || s.hi >= lim || (s.hi == -lim && s.lo == 0)) return false;
    *v = s.hi * 4294967296LL + (long long)s.lo;
    return true;
}

// status bits of the availability stage (f2) and of what is derived from it
enum : int {
    kFeErrInput = 1,        // |allocatable|, |overhead| or |a counted reservation| >= 2^61
    kFeErrResult = 2,       // a usage sum or an availability outside the exact-int64 domain
    kFeErrId = 4,           // resident forms: a reservation-table or overhead-table node id out of range or given twice
};

// The resident forms' directories: dir[id] = i for every node-table entry i with ids[i] != -1 (the directory is memset to -1
// first); atomicCAS from -1, so an id given twice is a refusal, not an overwrite.  Thread per entry of each of the two arrays
// (b_ids NULL: one).
__global__ void gp_resident_dirs(int32_t n, const int32_t* __restrict__ a_ids, int32_t a_lim, int32_t* __restrict__ a_dir,
                                 const int32_t* __restrict__ b_ids, int32_t b_lim, int32_t* __restrict__ b_dir, int* __restrict__ err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool bad = false;
    const int32_t a = a_ids[i];
    if (a != -1) bad |= a < 0 || a >= a_lim || atomicCAS(a_dir + a, -1, i) != -1;
    if (b_ids) {
        const int32_t b = b_ids[i];
        if (b != -1) bad |= b < 0 || b >= b_lim || atomicCAS(b_dir + b, -1, i) != -1;
    }
    if (bad) atomicOr(err, kFeErrId);
}

struct SortKey {          // 24 bytes
    long long mem;
    long long cpu;
    int az;               // AZ priority
    int name_rank;        // rank of the node name (unique)
};

__device__ __forceinline__ bool key_less(const SortKey& a, const SortKey& b) {
    if (a.az != b.az) return a.az < b.az;
    if (a.mem != b.mem) return a.mem < b.mem;
    if (a.cpu != b.cpu) return a.cpu < b.cpu;
    return a.name_rank < b.name_rank;
}

// per-zone totals of available memory / cpu (getAvailableResourcesByAZ, :124-134), exact whatever the node quantities:
// tot[4 * z ..] = memory (lo, hi), cpu (lo, hi) as exact_add keeps them
constexpr int kZoneTotWords = 4;
__device__ __forceinline__ void zone_total_add(unsigned long long* __restrict__ tot, int32_t z, long long mem, long long cpu) {
    unsigned long long* t = tot + (size_t)kZoneTotWords * z;
    exact_add(t + 0, t + 1, mem);
    exact_add(t + 2, t + 3, cpu);
}
// Instance groups (gp_prepare_cluster_zones_groups): ig[i] = the instance group of node i, -1 = none (NULL: every node in
// instance group 0).  Zones are then totalled and ranked per (instance group, zone) pair, pair = ig * n_zones + zone: a zone
// is ranked only against the zones of its own instance group, as PotentialNodes over that instance group's nodes ranks it.
__global__ void gp_zone_totals(int32_t n, const long long* __restrict__ cpu, const long long* __restrict__ mem,
                               const int32_t* __restrict__ zone, const int32_t* __restrict__ ig, int32_t n_zones,
                               unsigned long long* __restrict__ tot /* [kZoneTotWords * pairs] */) {
    int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t g = ig ? ig[i] : 0;
    if (g < 0) return;
    zone_total_add(tot, g * n_zones + zone[i], mem[i], cpu[i]);
}

// AZ priority = number of zones of the same instance group with smaller (mem, cpu, id)   (sort.Slice over zones, :102-104;
// ties by zone id); one thread per (instance group, zone) pair
__global__ void gp_zone_priority(int32_t n_pairs, int32_t n_zones, const unsigned long long* __restrict__ tot, int32_t* __restrict__ prio) {
    int32_t z = blockIdx.x * blockDim.x + threadIdx.x;
    if (z >= n_pairs) return;
    const unsigned long long* t = tot + (size_t)kZoneTotWords * z;
    const int32_t base = z - z % n_zones;
    z -= base;
    tot += (size_t)kZoneTotWords * base;
    const ExactSum m = exact_sum(t[0], t[1]), c = exact_sum(t[2], t[3]);
    int32_t p = 0;
    for (int32_t o = 0; o < n_zones; ++o) {
        const unsigned long long* u = tot + (size_t)kZoneTotWords * o;
        const ExactSum om = exact_sum(u[0], u[1]), oc = exact_sum(u[2], u[3]);
        const int by_mem = exact_cmp(om, m), by_cpu = exact_cmp(oc, c);
        const bool less = by_mem ? by_mem < 0 : (by_cpu ? by_cpu < 0 : o < z);
        p += less ? 1 : 0;
    }
    prio[base + z] = p;
}

// zone == NULL: one zone (priority 0, n_zones 1); name_rank == NULL: index order.  With instance groups the instance group
// is the leading key, folded into az = ig * n_zones + zone priority; nodes in no instance group sort last (az = n_ig *
// n_zones) and gp_split_candidates drops them.
__global__ void gp_make_keys(int32_t n, const long long* __restrict__ cpu, const long long* __restrict__ mem,
                             const int32_t* __restrict__ zone, const int32_t* __restrict__ zone_prio, const int32_t* __restrict__ ig,
                             int32_t n_ig, int32_t n_zones, const int32_t* __restrict__ name_rank, SortKey* __restrict__ keys) {
    int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SortKey k;
    const int32_t g = ig ? ig[i] : 0;
    k.mem = mem[i]; k.cpu = cpu[i];
    k.az = g < 0 ? n_ig * n_zones : g * n_zones + (zone ? zone_prio[g * n_zones + zone[i]] : 0);
    k.name_rank = name_rank ? name_rank[i] : i;
    keys[i] = k;
}

// ---- sort primitive (gangpack_tilesort.cuh): keys of this file ----------------------------------------------------
struct LabelKey {          // stable re-sort by label rank: (rank, position in the list) is unique
    uint32_t rank;
    int32_t pos;
};
__device__ __forceinline__ bool key_less(const LabelKey& a, const LabelKey& b) { return a.rank != b.rank ? a.rank < b.rank : a.pos < b.pos; }
// the label re-sort of instance-group-major candidate lists: stable within each instance group (seg), 12 bytes (a tile is
// exactly 48 KB, the default dynamic shared-memory limit)
struct SegLabelKey {
    uint32_t seg;
    uint32_t rank;
    int32_t pos;
};
__device__ __forceinline__ bool key_less(const SegLabelKey& a, const SegLabelKey& b) {
    return a.seg != b.seg ? a.seg < b.seg : (a.rank != b.rank ? a.rank < b.rank : a.pos < b.pos);
}
__device__ __forceinline__ SortKey key_max(const SortKey*) { SortKey k; k.mem = 0x7fffffffffffffffLL; k.cpu = 0x7fffffffffffffffLL; k.az = 0x7fffffff; k.name_rank = 0x7fffffff; return k; }
__device__ __forceinline__ LabelKey key_max(const LabelKey*) { LabelKey k; k.rank = 0xffffffffu; k.pos = 0x7fffffff; return k; }
__device__ __forceinline__ SegLabelKey key_max(const SegLabelKey*) { SegLabelKey k; k.seg = 0xffffffffu; k.rank = 0xffffffffu; k.pos = 0x7fffffff; return k; }

__global__ void gp_scatter_order(int32_t n, const int32_t* __restrict__ pos, int32_t* __restrict__ order) {
    int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) order[pos[i]] = i;
}

// Order-preserving compaction of the priority order into the driver and executor candidate lists (one CTA, every
// thread owns 8 consecutive positions per step).  counts[0] = #driver candidates, counts[1] = #executor candidates,
// counts[2] = #adjacent pairs of the order that the reference's comparator leaves undefined (same zone priority, memory
// and cpu but different gpu: SURVEY App. B6) -- 0 when no gpu column was given.  ig (NULL: one instance group): a node in
// no instance group is neither candidate nor part of a tie; ig_ties[g] (pre-zeroed, or NULL) counts instance group g's ties
// (the az key holds the instance group, so a tie never spans two).  IG: ig is given (the one-group call reads no ig).
constexpr int kSplitItems = 8;
template <bool IG>
__global__ void __launch_bounds__(1024) gp_split_candidates(int32_t n, const int32_t* __restrict__ order,
                                                            const uint8_t* __restrict__ is_candidate,
                                                            const uint8_t* __restrict__ unschedulable, const uint8_t* __restrict__ ready,
                                                            const SortKey* __restrict__ keys, const long long* __restrict__ gpu,
                                                            const int32_t* __restrict__ ig, int32_t* __restrict__ ig_ties,
                                                            int32_t* __restrict__ drv, int32_t* __restrict__ exe, int32_t* __restrict__ counts) {
    __shared__ int32_t wsum[2][32];
    __shared__ int32_t base[2];
    __shared__ int32_t ties;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (tid == 0) { base[0] = 0; base[1] = 0; ties = 0; }
    __syncthreads();
    int32_t my_ties = 0;
    for (int32_t p0 = 0; p0 < n; p0 += blockDim.x * kSplitItems) {
        const int32_t pb = p0 + tid * kSplitItems;
        int32_t node[kSplitItems];
        uint32_t fd = 0, fe = 0;
#pragma unroll
        for (int t = 0; t < kSplitItems; ++t) {
            const int32_t p = pb + t;
            node[t] = -1;
            if (p < n) {
                node[t] = order[p];
                const int32_t g = IG ? ig[node[t]] : 0;
                const uint32_t in = g >= 0 ? 1u : 0u;
                if (is_candidate ? is_candidate[node[t]] != 0 : true) fd |= in << t;
                if (!(unschedulable && unschedulable[node[t]]) && (ready ? ready[node[t]] != 0 : true)) fe |= in << t;
                if (in && gpu && p > 0) {
                    const int32_t prev = t > 0 ? node[t - 1] : order[p - 1];
                    const SortKey a = keys[prev], b = keys[node[t]];
                    if (a.az == b.az && a.mem == b.mem && a.cpu == b.cpu && gpu[prev] != gpu[node[t]]) {
                        ++my_ties;
                        if (IG) atomicAdd(ig_ties + g, 1);
                    }
                }
            }
        }
        const int32_t cd = __popc(fd), ce = __popc(fe);
        // exclusive scan of (cd, ce) over the block
        int32_t id = cd, ie = ce;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int32_t ud = __shfl_up_sync(0xffffffffu, id, d), ue = __shfl_up_sync(0xffffffffu, ie, d);
            if (lane >= d) { id += ud; ie += ue; }
        }
        if (lane == 31) { wsum[0][w] = id; wsum[1][w] = ie; }
        __syncthreads();
        int32_t od = base[0] + id - cd, oe = base[1] + ie - ce;
        for (int k = 0; k < w; ++k) { od += wsum[0][k]; oe += wsum[1][k]; }
#pragma unroll
        for (int t = 0; t < kSplitItems; ++t) {
            if (fd & (1u << t)) drv[od++] = node[t];
            if (fe & (1u << t)) exe[oe++] = node[t];
        }
        __syncthreads();
        if (tid == 0) {
            int32_t td = 0, te = 0;
            for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { td += wsum[0][k]; te += wsum[1][k]; }
            base[0] += td; base[1] += te;
        }
        __syncthreads();
    }
    if (my_ties) atomicAdd(&ties, my_ties);
    __syncthreads();
    if (tid == 0) { counts[0] = base[0]; counts[1] = base[1]; counts[2] = ties; }
}

// Stable re-sort of a candidate list by label rank (createLabelLessThanFunction :161-180: unknown rank sorts
// last, ties keep their order): keys (rank, position) through the sort primitive above, then out[pos_i] = list[i].
__global__ void gp_label_keys(const int32_t* __restrict__ count_ptr, const int32_t* __restrict__ list,
                              const int32_t* __restrict__ label_rank, LabelKey* __restrict__ keys) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count_ptr) return;
    const int32_t lr = label_rank[list[i]];
    LabelKey k; k.rank = lr < 0 ? 0x7fffffffu : (uint32_t)lr; k.pos = i;
    keys[i] = k;
}
// the same within each instance group: (ig, rank, position)
__global__ void gp_seg_label_keys(const int32_t* __restrict__ count_ptr, const int32_t* __restrict__ list,
                                  const int32_t* __restrict__ label_rank, const int32_t* __restrict__ ig, SegLabelKey* __restrict__ keys) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count_ptr) return;
    const int32_t v = list[i], lr = label_rank[v];
    SegLabelKey k; k.seg = (uint32_t)ig[v]; k.rank = lr < 0 ? 0x7fffffffu : (uint32_t)lr; k.pos = i;
    keys[i] = k;
}
__global__ void gp_label_scatter(const int32_t* __restrict__ count_ptr, const int32_t* __restrict__ list,
                                 const int32_t* __restrict__ pos, int32_t* __restrict__ out) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < *count_ptr) out[pos[i]] = list[i];
}

// ---- SURVEY 8f row f2: the availability snapshot from reservations -------------------------------------------
// usage[node] = sum of the resources of every (hard or soft) reservation on that node: UsageForNodes
// (LIB/resources/resources.go:31-43) + UsedSoftReservationResources (internal/cache/softreservations.go:155-170),
// summed as in GetReservedResources (EXT/resourcereservations.go:258-263).  A segmented reduction over
// (reservation -> node) pairs: thread per reservation, exact_add per dimension (integer adds commute: exact, and no
// sum wraps).  usage[(2 * d + half) * n_nodes + node]: dimension d, half 0 = lo, 1 = hi.
// Where finds the node-table index of row r (-1: the row is not counted): UsageRowIndex for the per-call rows, UsageSlotDir for
// the slots of the resident reservation table.
struct UsageRowIndex {                  // gp_usage_input.res_node: an index outside [0, n_nodes) is not in the list
    const int32_t* res_node;
    int32_t n_nodes;
    __device__ int32_t operator()(long long r) const {
        const int32_t node = res_node[r];
        return node < 0 || node >= n_nodes ? -1 : node;
    }
};
struct UsageSlotDir {                   // a slot's node id through the per-call directory (node id -> node-table index, -1 = none)
    const int32_t* slot_node;           // [n_slots] -1 = free slot; occupied slots hold ids in [0, n_node_ids), checked when written
    const int32_t* dir;                 // [n_node_ids]
    __device__ int32_t operator()(long long r) const {
        const int32_t id = slot_node[r];
        return id < 0 ? -1 : dir[id];
    }
};
template <class Where>
__global__ void gp_usage_scatter(long long n_res, Where where, const long long* __restrict__ res_cpu,
                                 const long long* __restrict__ res_mem, const long long* __restrict__ res_gpu, int32_t n_nodes,
                                 unsigned long long* __restrict__ usage /* [6][n_nodes] */, unsigned int* __restrict__ has_entry /* [n_nodes] or NULL */,
                                 int* __restrict__ err) {
    const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (r >= n_res) return;
    const int32_t node = where(r);
    if (node < 0) return;                               // reservation on a node that is not in the list: ignored (:67-75)
    if (has_entry) has_entry[node] = 1u;                // the usage map has an entry for this node (whatever its value)
    const long long v[3] = {res_cpu[r], res_mem[r], res_gpu ? res_gpu[r] : 0};
    const size_t N = (size_t)n_nodes;
    bool bad = false;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        bad |= !in_domain(v[d]);
        exact_add(usage + (size_t)(2 * d) * N + node, usage + (size_t)(2 * d + 1) * N + node, v[d]);
    }
    if (bad) atomicOr(err, kFeErrInput);
}

// NodeSchedulingMetadataForNodes (resources.go:61-100): available = allocatable - (usage + overhead),
// schedulable = allocatable - overhead.  Inputs and usage sums inside the domain keep every expression below 2^63, so
// nothing wraps before it is checked; whatever leaves the domain is reported in *err and the rows written are then not results.
__global__ void gp_availability(int32_t n, const long long* __restrict__ alloc_cpu, const long long* __restrict__ alloc_mem,
                                const long long* __restrict__ alloc_gpu, const long long* __restrict__ over_cpu,
                                const long long* __restrict__ over_mem, const long long* __restrict__ over_gpu,
                                const unsigned long long* __restrict__ usage /* [6][n] */, long long* __restrict__ avail /* [3][n] */,
                                long long* __restrict__ sched /* [3][n] */, int* __restrict__ err,
                                const unsigned int* __restrict__ has_entry = nullptr, long long* __restrict__ resched /* [3][n] or NULL */ = nullptr) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long a[3] = {alloc_cpu[i], alloc_mem[i], alloc_gpu ? alloc_gpu[i] : 0};
    const long long o[3] = {over_cpu ? over_cpu[i] : 0, over_mem ? over_mem[i] : 0, over_gpu ? over_gpu[i] : 0};
    int bad = 0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        long long u = 0, av = 0, sc = 0, rs = 0;
        if (!in_domain(a[d]) || !in_domain(o[d])) bad |= kFeErrInput;
        else if (!exact_value(exact_sum(usage[(size_t)(2 * d) * n + i], usage[(size_t)(2 * d + 1) * n + i]), &u)) bad |= kFeErrResult;
        else {
            av = a[d] - (u + o[d]);
            sc = a[d] - o[d];
            // availableResources of rescheduleExecutor (EXT/resource.go:638-643): NodeSchedulingMetadataForNodes has already added
            // the overhead into the usage map's EXISTING entries in place when usage.Add(overhead) adds it again (SURVEY App. B7)
            rs = resched ? a[d] - (u + o[d] * (has_entry[i] ? 2 : 1)) : 0;
            if (!in_domain(av) || !in_domain(sc) || !in_domain(rs)) bad |= kFeErrResult;
        }
        avail[(size_t)d * n + i] = av;
        sched[(size_t)d * n + i] = sc;
        if (resched) resched[(size_t)d * n + i] = rs;
    }
    if (bad) atomicOr(err, bad);
}

}  // namespace gp

// gangpack_placement.cuh -- the driver Predicate's placement metrics on the device: driver-executor collocation, executor node
// count and cross-zone pod pairs (gp_placement_metrics[_device]).
//
// Reference (EXT = internal/extender, MET = internal/metrics):
//   selectDriverNode, after a successful pack                EXT/resource.go:352-357
//   ReportInitialDriverExecutorCollocationMetric             MET/metrics.go:223-252
//   ReportInitialNodeCountMetrics                            MET/metrics.go:254-275
//   ReportCrossZoneMetric / crossZoneTraffic                 MET/metrics.go:277-318, 322-330
//
// Per placed row (driver d, ExecutorNodes e[0..k)): E = {e_t}, collocation from d in E and |E|, k / |E|, and the pod histogram
// over the zones: c_z = pods on in-scope nodes of metric zone z, the driver's node counting one pod more.  crossZoneTraffic
// is T*S - (S^2 + sum c_z^2) / 2 with T = k + 1 and S = sum c_z (DESIGN §2.8), so the kernel needs only S, sum c_z^2 and the
// number of non-empty zones -- never the map.  The executor order is not relied on (node-major, round-major, capacity order
// or a zone result alike).
//
// One team per row.  Its slice is a node bitmap ([ceil(n_nodes / 32)] words: the first atomicOr setter of a bit counts a
// distinct node) and one counter per metric zone (an atomicAdd that returns o adds 2o + 1 to sum c_z^2 and, for o == 0, one
// zone).  The team walks the row a second time to clear exactly what it set, so a slice is zeroed once per kernel, not per
// row.  Rows of up to kPmLongRow executors take a warp (gp_placement_rows<false>, several warps per CTA); a placed row above
// that is listed by the warp kernel and taken by a whole CTA (gp_placement_rows<true>).  Slices live in dynamic shared
// memory when they fit (about 1.8 M nodes without zones), in global scratch otherwise.  Each record is written once, by its
// row's team; the status word and the long-row list are the only atomics.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "gangpack.h"

namespace gp {

constexpr int kPmThreads = 256;                 // threads of a CTA team (and of the warp kernel's CTA at most)
constexpr int32_t kPmLongRow = 2048;            // placed rows with more executor entries take a CTA
constexpr int kPmErrNode = 1;                   // a placed row's driver or executor node outside [0, n_nodes)
constexpr int kPmErrZone = 2;                   // a metric zone outside [0, n_metric_zones)
constexpr int kPmErrGroup = 4;                  // an instance_group value outside [-1, G) or a row's group outside [0, G)
constexpr int kPmErrCount = 8;                  // a negative exe_count
constexpr int kPmErrCapacity = 16;              // a placed row's ExecutorNodes range outside [0, executor_nodes_cap)
constexpr int kPmErrUnrepresentable = 32;       // an exe_count above 2^24 (the gp_apps bound that keeps every value exact)
constexpr int32_t kPmMaxCount = 1 << 24;

// [0] status bits, [1] long rows listed: zeroed by a memset at the start of every call
struct PmState { int err; unsigned int n_long; };

struct PmIn {
    const int32_t* count;            // exe_count [n_apps]
    const int64_t* off;              // [n_apps + 1] ExecutorNodes offsets
    const int32_t* group;            // [n_apps] or NULL (= 0); read only with ig
    const int32_t* driver;           // [n_apps]
    const int32_t* exec;             // [cap]
    long long cap;
    const int32_t* zone;             // [n_nodes] metric zone
    const int32_t* ig;               // [n_nodes] instance group, -1 = none; NULL: every node in scope
    int32_t n_apps, n_nodes, n_zones, n_ig;
    int32_t bitmap_words;
    long long slice_words;           // bitmap words + n_zones counters
    uint32_t* gslices;               // global-scratch slices (one per team), or NULL: slices in dynamic shared memory
    int32_t* long_rows;              // [n_apps] rows for the CTA kernel
    PmState* state;
};

__device__ __forceinline__ bool pm_long_row(int32_t d, int32_t k) { return d >= 0 && k > kPmLongRow; }

template <bool CTA> __device__ __forceinline__ void pm_team_sync() {
    if (CTA) __syncthreads(); else __syncwarp();
}

// sums over the team; every member ends with them (CTA: through `part`, blockDim.x / 32 entries)
struct PmSums { int32_t distinct, zones, pods, hosts, bad; long long sq; };

__device__ __forceinline__ PmSums pm_warp_sum(PmSums s) {
    s.distinct = (int32_t)__reduce_add_sync(0xffffffffu, (unsigned)s.distinct);
    s.zones = (int32_t)__reduce_add_sync(0xffffffffu, (unsigned)s.zones);
    s.pods = (int32_t)__reduce_add_sync(0xffffffffu, (unsigned)s.pods);
    s.hosts = (int32_t)__reduce_or_sync(0xffffffffu, (unsigned)s.hosts);
    s.bad = (int32_t)__reduce_or_sync(0xffffffffu, (unsigned)s.bad);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s.sq += __shfl_xor_sync(0xffffffffu, s.sq, o);
    return s;
}

template <bool CTA> __device__ __forceinline__ PmSums pm_team_sum(PmSums s, PmSums* part) {
    s = pm_warp_sum(s);
    if (!CTA) return s;
    const int warps = blockDim.x >> 5;
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    PmSums t = part[0];
    for (int w = 1; w < warps; ++w) {
        const PmSums& u = part[w];
        t.distinct += u.distinct; t.zones += u.zones; t.pods += u.pods; t.hosts |= u.hosts; t.bad |= u.bad; t.sq += u.sq;
    }
    __syncthreads();                 // part is reused by the next row
    return t;
}

// one placed row by one team of `size` threads, member r; slice = [bitmap | zone counters], zero on entry and on return
template <bool CTA>
__device__ __forceinline__ void pm_row(const PmIn& in, int32_t i, int32_t d, int32_t k, uint32_t* slice, int r, int size, PmSums* part,
                                       gp_placement_record* __restrict__ out) {
    uint32_t* bm = slice;
    uint32_t* cz = slice + in.bitmap_words;
    const int32_t g = in.ig && in.group ? in.group[i] : 0;
    const int32_t* ex = in.exec + in.off[i];
    PmSums s{0, 0, 0, 0, 0, 0};
    // pass 1: t < k the executor entries, t == k the driver's own pod
    for (int32_t t = r; t <= k; t += size) {
        const int32_t n = t < k ? ex[t] : d;
        if (n < 0 || n >= in.n_nodes) { s.bad |= kPmErrNode; continue; }
        if (t < k) {
            s.hosts |= n == d;
            const uint32_t bit = 1u << (n & 31);
            if (!(atomicOr(&bm[n >> 5], bit) & bit)) ++s.distinct;
        }
        if (in.ig && in.ig[n] != g) continue;                  // outside availableNodes: in T, in no zone
        const int32_t z = in.zone[n];
        if (z < 0 || z >= in.n_zones) { s.bad |= kPmErrZone; continue; }
        const uint32_t o = atomicAdd(&cz[z], 1u);
        s.sq += 2ll * o + 1;
        s.zones += o == 0u;
        ++s.pods;
    }
    pm_team_sync<CTA>();
    // pass 2: clear what pass 1 set (a bitmap word holds only this row's bits, so the whole word goes)
    for (int32_t t = r; t <= k; t += size) {
        const int32_t n = t < k ? ex[t] : d;
        if (n < 0 || n >= in.n_nodes) continue;
        if (t < k) bm[n >> 5] = 0u;
        if (in.ig && in.ig[n] != g) continue;
        const int32_t z = in.zone[n];
        if (z >= 0 && z < in.n_zones) cz[z] = 0u;
    }
    pm_team_sync<CTA>();
    s = pm_team_sum<CTA>(s, part);
    if (r != 0) return;
    gp_placement_record m{-1, 0, 0, 0, 0, 0};
    if (s.bad) {
        atomicOr(&in.state->err, s.bad);
    } else {
        const long long T = (long long)k + 1, S = s.pods;
        m.collocation = !s.hosts ? 0 : s.distinct == 1 ? 1 : 2;
        m.distinct_exec_nodes = s.distinct;
        m.execs_per_node = k > 0 ? k / s.distinct : -1;
        m.n_zones = s.zones;
        m.cross_zone_pairs = T * S - (S * S + s.sq) / 2;
        m.total_pairs = T * (T - 1) / 2;
    }
    out[i] = m;
}

// CTA == false: warps over every row (the node-column checks first, grid-stride); a placed row above kPmLongRow is listed for
// the CTA kernel.  CTA == true: one CTA per listed row.
template <bool CTA>
__global__ void __launch_bounds__(kPmThreads) gp_placement_rows(PmIn in, gp_placement_record* __restrict__ out) {
    extern __shared__ uint32_t pm_smem[];
    __shared__ PmSums part[kPmThreads / 32];
    const int size = CTA ? (int)blockDim.x : 32;
    const int teams = CTA ? 1 : (int)(blockDim.x >> 5);
    const int team = CTA ? 0 : (int)(threadIdx.x >> 5);
    const int r = CTA ? (int)threadIdx.x : (int)(threadIdx.x & 31);
    const long long tid = (long long)blockIdx.x * teams + team, n_teams = (long long)gridDim.x * teams;
    uint32_t* slice = in.gslices ? in.gslices + (size_t)tid * (size_t)in.slice_words : pm_smem + (size_t)team * (size_t)in.slice_words;
    for (int32_t w = r; w < in.slice_words; w += size) slice[w] = 0u;
    pm_team_sync<CTA>();
    if (!CTA) {
        int bad = 0;
        for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < in.n_nodes; v += (long long)gridDim.x * blockDim.x) {
            const int32_t z = in.zone[v];
            if (z < 0 || z >= in.n_zones) bad |= kPmErrZone;
            if (in.ig && (in.ig[v] < -1 || in.ig[v] >= in.n_ig)) bad |= kPmErrGroup;
        }
        if (bad) atomicOr(&in.state->err, bad);
        for (long long i = tid; i < in.n_apps; i += n_teams) {
            const int32_t d = in.driver[i], k = in.count[i];
            int bad_row = 0;
            if (k < 0) bad_row |= kPmErrCount;
            if (k > kPmMaxCount) bad_row |= kPmErrUnrepresentable;
            if (in.ig && in.group && (in.group[i] < 0 || in.group[i] >= in.n_ig)) bad_row |= kPmErrGroup;
            if (d >= in.n_nodes) bad_row |= kPmErrNode;
            if (d >= 0 && k >= 0 && (in.off[i] < 0 || in.off[i] > in.cap - k)) bad_row |= kPmErrCapacity;
            if (d >= 0 && !bad_row && pm_long_row(d, k)) {
                if (r == 0) in.long_rows[atomicAdd(&in.state->n_long, 1u)] = (int32_t)i;
                continue;
            }
            if (d < 0 || bad_row) {                                // not reported (or refused: the record is not used)
                if (r == 0) {
                    if (bad_row) atomicOr(&in.state->err, bad_row);
                    out[i] = gp_placement_record{-1, 0, 0, 0, 0, 0};
                }
                continue;
            }
            pm_row<false>(in, (int32_t)i, d, k, slice, r, size, part, out);
        }
    } else {
        const unsigned int n_long = in.state->n_long;              // the warp kernel has ended (stream order)
        for (unsigned int j = blockIdx.x; j < n_long; j += gridDim.x) {
            const int32_t i = in.long_rows[j];
            pm_row<true>(in, i, in.driver[i], in.count[i], slice, r, size, part, out);
        }
    }
}

// after both row kernels: the status the call returns (GP_OK / GP_ERR_INVALID / GP_ERR_UNREPRESENTABLE / GP_ERR_CAPACITY) to
// *status and the bits to *bits (either may be NULL)
__global__ void gp_placement_finish(const PmState* __restrict__ state, int32_t* __restrict__ status, int32_t* __restrict__ bits) {
    if (threadIdx.x != 0) return;
    const int e = state->err;
    if (status)
        *status = e & ~(kPmErrCapacity | kPmErrUnrepresentable) ? GP_ERR_INVALID : e & kPmErrUnrepresentable ? GP_ERR_UNREPRESENTABLE
                  : e ? GP_ERR_CAPACITY : GP_OK;
    if (bits) *bits = e;
}

// device form without exec_out_off: off[0..n] = the exclusive prefix sum of max(exe_count, 0), one CTA of kPmThreads
__global__ void __launch_bounds__(kPmThreads) gp_placement_offsets(const int32_t* __restrict__ count, int32_t n, int64_t* __restrict__ off) {
    __shared__ long long part[kPmThreads];
    const int32_t per = (n + kPmThreads - 1) / kPmThreads;
    const int32_t lo = min(n, (int32_t)threadIdx.x * per), hi = min(n, lo + per);
    long long s = 0;
    for (int32_t i = lo; i < hi; ++i) s += count[i] > 0 ? count[i] : 0;
    part[threadIdx.x] = s;
    __syncthreads();
    for (int o = 1; o < kPmThreads; o <<= 1) {                 // inclusive Hillis-Steele scan of the chunk sums
        const long long v = threadIdx.x >= (unsigned)o ? part[threadIdx.x - o] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    long long acc = part[threadIdx.x] - s;
    for (int32_t i = lo; i < hi; ++i) { off[i] = acc; acc += count[i] > 0 ? count[i] : 0; }
    if (threadIdx.x == kPmThreads - 1) off[n] = part[kPmThreads - 1];
}

}  // namespace gp

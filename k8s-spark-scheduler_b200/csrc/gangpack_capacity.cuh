// gangpack_capacity.cuh -- the unschedulable-pod marker's capacity checks on the device, for every `binpack:` packer.
//
// Reference (EXT = internal/extender, LIB = vendor/github.com/palantir/k8s-spark-scheduler-lib/pkg):
//   scanForUnschedulablePods / DoesPodExceedClusterCapacity   EXT/unschedulablepods.go:93-166
//   NodeSchedulingMetadataForNodes (zero usage)               LIB/resources/resources.go:61-100
//   SparkBinPack + the five packers                           LIB/binpack/*.go
//
// Every stale driver is packed against zero usage, with its affinity nodes in lister order as both priority orders.  DESIGN
// §2.2 proves that the answer needs neither that order nor a placement: with cap(n|r) the executor capacity of DESIGN §2,
// C = 2^31 and, over the driver's node set (or one zone of it),
//   T = sum_n min(cap(n|0), C)      M = max over nodes d the driver fits on of min(cap(d|drv), C) - min(cap(d|0), C)
// the pack succeeds iff a driver fits and T + M >= exe_count, for tightly-pack, distribute-evenly and minimal-fragmentation
// alike; az-aware-tightly-pack is that over the whole set; the two single-AZ packers need it in one zone and a positive
// average packing efficiency, which under zero usage depends on the requests alone.
//
// A driver's node set is a class.  Two layouts of the classes:
//   gp_exceeds_cluster_capacity           one class per node (node_group) plus the class of every node, for class -1 drivers:
//                                         entry k = 0 of node i is its class, k = 1 the all-nodes class (slot G);
//   gp_exceeds_cluster_capacity_affinity  class a = the nodes affinity a matches (gangpack_affinity.cuh), any subsets of the
//                                         nodes, overlapping freely: entry k of node i is affinity a0 + k when it matches.
// The entries of one chunk of classes are (k, node) for k < K; K x n_nodes stays below kCapEntries, so the scratch is bounded
// whatever the number of memberships: more affinities take more chunks, never a refusal.  The pair results are kept across
// chunks; each chunk resets and fills only the pairs of its own classes.
//
// Kernels (one stream, no host round trip between them):
//   gp_cc_nodes        thread per node: validate, schedulable = alloc - overhead, zone
//   gp_cc_intern       thread per driver: validate, intern (class, executor shape, driver shape) -> dense pair id
//   per chunk of classes [a0, a0 + K):
//     gp_cc_keys         thread per entry: its bucket (class k, zone), -1 = the node is not in class k
//     gp_cc_bucket_scan  one CTA: node, segment and multi-segment offsets of the buckets
//     gp_cc_scatter      thread per entry: nodes grouped by bucket; the first node of every segment writes the segment
//     gp_cc_pair_scan    one CTA: prefix over the pairs of the number of segments each one visits; the chunk's pairs reset
//     per chunk of pairs (one chunk unless pairs x multi-segment buckets exceed kCapSlotEntries):
//       gp_cc_clear      zero the chunk's (pair, multi-segment bucket) slots
//       gp_cc_pass       CTA per (pair, segment): T and M of the segment, warp -> CTA -> global atomics on the pair; a zone's
//                        T_z + M_z is complete in the CTA that holds its only segment, or in the last of its segments to arrive
//   gp_cc_decide       thread per driver: O(1)
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "gangpack_kernels.cuh"

namespace gp {

constexpr int kCapThreads = 256;
constexpr int32_t kCapSeg = 16 * kCapThreads;         // nodes of one bucket per work item of the pass
constexpr uint32_t kCapClamp = 1u << 31;               // C: above every int32 exe_count
constexpr long long kCapNone = -0x7fffffffffffffffLL - 1;         // INT64_MIN: "no driver fits"
// Scratch bound: a bucket of more than kCapSeg nodes is split over several CTAs, which combine its (T_z, M_z) in a slot per
// (pair, such bucket).  There are at most K n_nodes / (kCapSeg + 1) such buckets in a chunk of K classes, whatever the number of zones; a chunk of
// pairs owns at most kCapSlotEntries slots (24 bytes each, 48 MiB in all), more pairs take more chunks, never a refusal.
constexpr int64_t kCapSlotEntries = (int64_t)1 << 21;
// Entries of one chunk of affinity classes (K x n_nodes, 32 bytes each: 64 MiB); one chunk holds at least one class.
constexpr int64_t kCapEntries = (int64_t)1 << 21;

enum : int {
    kCcErrNegative = 1,         // negative request or exe_count
    kCcErrUnrepresentable = 2,  // request >= 2^61
    kCcErrGroup = 4,            // driver class outside [-1, n_groups)
    kCcErrZone = 8,             // zone_id outside [0, n_zones)
    kCcErrNodeGroup = 16,       // node_group outside [-1, n_groups)
    kCcErrNodeQuantity = 32,    // |allocatable| or |overhead| >= 2^61
};

// One interned (class, executor shape, driver shape): the division recipes of the executor request and the driver request
struct CapPair {
    DimDiv div[3];
    long long drv[3];
    int32_t cls;                // -1: every node
    int32_t pad;
};

// Open-addressing entry: key = fingerprint (0 = empty), the full tuple, published by `ready`
struct CapEntry {
    unsigned long long key;
    long long q[6];             // drv cpu, mem, gpu, exe cpu, mem, gpu
    int32_t group;
    int32_t id;
    int32_t ready;
    int32_t pad;
};

struct CapNodesIn {
    int32_t n;
    const long long* alloc[3];
    const long long* over[3];   // NULL = 0
    const int32_t* zone;        // NULL = zone 0
    const int32_t* group;       // NULL = class 0
};

// The classes of one chunk: member == NULL -> node_group classes (K = 2), else the affinity bitmap of gangpack_affinity.cuh
struct CapClassesIn {
    const int32_t* group;       // [n] node_group, NULL = class 0
    const uint32_t* member;     // [K][words]: row k = affinity a0 + k
    int32_t words;
};

// kCapSeg consecutive nodes (or fewer, at the end) of one bucket
struct CapSeg {
    int32_t first, len;
    int32_t nseg;               // segments of the bucket
    int32_t ms;                 // index of the bucket among those with nseg > 1, -1 = a single segment
};

struct CapScratch {
    int32_t* key;               // [K n] entry k n + i: node i's bucket in class k of the chunk, -1 = not in it (or invalid)
    int32_t* rank;              // [K n] the node's position in that bucket
    int32_t* zone;              // [n] the node's zone, -1 = invalid node
    int32_t* bucket_cnt;        // [B]
    int32_t* bucket_off;        // [B + 1]
    int32_t* seg_off;           // [B + 1]
    int32_t* ms_off;            // [B + 1]
    long long* staged[3];       // [n] schedulable resources in node-table order
    long long* sched[3];        // [K n] the same, nodes grouped by bucket (once per class of the chunk it is in)
    CapSeg* segs;               // [n_segs]
    int* err;
    int32_t B, Z, G, n;
    int32_t K;                  // classes in the chunk: 2 for node_group (slot G = every node), <= n_aff for affinities
    int32_t a0;                 // affinity layout: the chunk's first class; -1 = node_group layout
};

// (pair, multi-segment bucket): the bucket's partial T_z and M_z, and how many of its segments have added theirs
struct CapSlot {
    unsigned long long sum;
    long long mx;
    unsigned int arrived;
    int pad;
};

__device__ __forceinline__ unsigned long long warp_sum64(unsigned long long v) {
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(kFull, v, d);
    return v;
}
__device__ __forceinline__ long long warp_max64(long long v) {
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) v = max(v, (long long)__shfl_xor_sync(kFull, v, d));
    return v;
}

// Exclusive scan of one value per thread of a 1024-thread CTA; *total = the CTA's sum.  Every thread must call it.
__device__ __forceinline__ long long cta_excl_scan(long long v, long long* sh /* [32] */, long long* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    long long inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const long long t = __shfl_up_sync(kFull, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) sh[w] = inc;
    __syncthreads();
    if (w == 0) {
        long long s = sh[lane], si = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long t = __shfl_up_sync(kFull, si, d);
            if (lane >= d) si += t;
        }
        sh[lane] = si - s;
        if (lane == 31) sh[32] = si;
    }
    __syncthreads();
    const long long r = sh[w] + inc - v;
    *total = sh[32];
    __syncthreads();
    return r;
}

// ---- nodes --------------------------------------------------------------------------------------------------------
__global__ void gp_cc_nodes(CapNodesIn in, CapScratch s) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= in.n) return;
    int bad = 0;
    long long v[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const long long a = in.alloc[d] ? in.alloc[d][i] : 0, o = in.over[d] ? in.over[d][i] : 0;
        if (a >= kMaxQuantity || a <= -kMaxQuantity || o >= kMaxQuantity || o <= -kMaxQuantity) bad |= kCcErrNodeQuantity;
        v[d] = a - o;                                  // SchedulableResources = AvailableResources under zero usage
    }
    const int32_t z = in.zone ? in.zone[i] : 0;
    const int32_t g = in.group ? in.group[i] : 0;
    if (z < 0 || z >= s.Z) bad |= kCcErrZone;
    if (in.group && (g < -1 || g >= s.G)) bad |= kCcErrNodeGroup;     // NULL: every node in class 0
    if (bad) { atomicOr(s.err, bad); s.zone[i] = -1; return; }
    s.zone[i] = z;
#pragma unroll
    for (int d = 0; d < 3; ++d) s.staged[d][i] = v[d];
}

// entry j = k n + i: node i in class k of the chunk -> bucket k Z + zone
__global__ void gp_cc_keys(CapClassesIn in, CapScratch s) {
    const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (j >= (long long)s.K * s.n) return;
    const int32_t k = (int32_t)(j / s.n), i = (int32_t)(j - (long long)k * s.n), z = s.zone[i];
    int32_t cls;                // the entry's bucket row, -1 = node i is not in class k
    if (in.member) cls = (in.member[(long long)k * in.words + (i >> 5)] >> (i & 31)) & 1u ? k : -1;
    else if (k == 1) cls = s.G;  // class slot G holds every node by zone: a class -1 driver's zone is one bucket
    else cls = in.group ? in.group[i] : 0;
    const int32_t key = z >= 0 && cls >= 0 ? cls * s.Z + z : -1;
    s.key[j] = key;
    if (key >= 0) s.rank[j] = atomicAdd(s.bucket_cnt + key, 1);
}

__global__ void __launch_bounds__(1024) gp_cc_bucket_scan(CapScratch s) {
    __shared__ long long sh[33];
    long long nbase = 0, sbase = 0, mbase = 0;
    for (int32_t b0 = 0; b0 < s.B; b0 += 1024) {
        const int32_t b = b0 + (int32_t)threadIdx.x;
        const long long cnt = b < s.B ? s.bucket_cnt[b] : 0;
        long long ntot, stot, mtot;
        const long long ne = cta_excl_scan(cnt, sh, &ntot);
        const long long se = cta_excl_scan((cnt + kCapSeg - 1) / kCapSeg, sh, &stot);
        const long long me = cta_excl_scan(cnt > kCapSeg ? 1 : 0, sh, &mtot);
        if (b < s.B) { s.bucket_off[b] = (int32_t)(nbase + ne); s.seg_off[b] = (int32_t)(sbase + se); s.ms_off[b] = (int32_t)(mbase + me); }
        nbase += ntot; sbase += stot; mbase += mtot;
    }
    if (threadIdx.x == 0) { s.bucket_off[s.B] = (int32_t)nbase; s.seg_off[s.B] = (int32_t)sbase; s.ms_off[s.B] = (int32_t)mbase; }
}

__global__ void gp_cc_scatter(CapScratch s) {
    const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;     // entry k n + i
    if (j >= (long long)s.K * s.n) return;
    const int32_t key = s.key[j], i = (int32_t)(j % s.n);
    if (key < 0) return;
    const int32_t r = s.rank[j], pos = s.bucket_off[key] + r;
    s.sched[0][pos] = s.staged[0][i]; s.sched[1][pos] = s.staged[1][i]; s.sched[2][pos] = s.staged[2][i];
    if (r % kCapSeg == 0) {
        const int32_t cnt = s.bucket_cnt[key];
        CapSeg sg;
        sg.first = pos; sg.len = min(kCapSeg, cnt - r); sg.nseg = (cnt + kCapSeg - 1) / kCapSeg;
        sg.ms = cnt > kCapSeg ? s.ms_off[key] : -1;
        s.segs[s.seg_off[key] + r / kCapSeg] = sg;
    }
}

// ---- drivers: validate and intern ---------------------------------------------------------------------------------
struct CapAppsIn {
    int32_t n;
    const long long* q[6];      // drv cpu, mem, gpu, exe cpu, mem, gpu (gpu columns NULL = 0)
    const int32_t* count;
    const int32_t* group;       // NULL = class 0
    int32_t n_groups;
    int32_t min_group;          // -1: node_group classes (-1 = every node); 0: affinity ids
    uint32_t hash_mask;         // table size - 1; the size is a power of two >= 2 n
};

__device__ __forceinline__ int ld_acquire_i32(const int32_t* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// One lane per distinct fingerprint of a warp probes; an entry whose fingerprint matches is used only once its full tuple
// is published and equal, so a collision costs a probe, never a wrong answer.  The table has more slots than drivers: a
// probe always ends.
__device__ __forceinline__ int32_t cc_intern(CapEntry* table, uint32_t mask, unsigned long long fp, const long long* q, int32_t g,
                                             CapPair* pairs, int32_t* n_pairs) {
    uint32_t slot = (uint32_t)fp & mask;
    for (;;) {
        CapEntry* en = table + slot;
        unsigned long long cur = atomicCAS(&en->key, 0ull, fp);
        if (cur == 0ull) {                              // claimed: fill, number, publish
            for (int t = 0; t < 6; ++t) en->q[t] = q[t];
            en->group = g;
            const int32_t id = atomicAdd(n_pairs, 1);
            en->id = id;
            CapPair p;
            int bad = 0; uint64_t l; bool fast = true;
            for (int d = 0; d < 3; ++d) { p.div[d] = prep_dim(0, q[3 + d], d, 0, bad, l, fast); p.drv[d] = q[d]; }
            p.cls = g; p.pad = 0;
            pairs[id] = p;
            __threadfence();
            atomicExch(&en->ready, 1);
            return id;
        }
        if (cur == fp) {
            unsigned ns = 32;
            while (ld_acquire_i32(&en->ready) == 0) { __nanosleep(ns); if (ns < 512) ns <<= 1; }
            const volatile CapEntry* ve = en;
            bool same = ve->group == g;
            for (int t = 0; t < 6; ++t) same = same && ve->q[t] == q[t];
            if (same) return ve->id;
        }
        slot = (slot + 1) & mask;
    }
}

__global__ void gp_cc_intern(CapAppsIn in, CapEntry* table, CapPair* pairs, int32_t* n_pairs, int32_t* app_pair, int* err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const unsigned act = __ballot_sync(kFull, i < in.n);
    if (i >= in.n) return;
    long long q[6];
    int bad = 0;
#pragma unroll
    for (int t = 0; t < 6; ++t) {
        q[t] = in.q[t] ? in.q[t][i] : 0;
        if (q[t] < 0) bad |= kCcErrNegative;
        if (q[t] >= kMaxQuantity) bad |= kCcErrUnrepresentable;
    }
    if (in.count[i] < 0) bad |= kCcErrNegative;
    const int32_t g = in.group ? in.group[i] : 0;
    if (g < in.min_group || g >= in.n_groups) bad |= kCcErrGroup;
    if (bad) atomicOr(err, bad);
    // chained, so that no exchange of fields between the two shapes or the class leaves the fingerprint unchanged
    unsigned long long fp = shape_fingerprint(q[3], q[4], q[5]);
    fp = shape_fingerprint((long long)fp, q[0], q[1]);
    fp = shape_fingerprint((long long)fp, q[2], (long long)g);
    // The lanes that share a fingerprint elect one leader to probe; a lane takes the leader's pair only when its full tuple
    // equals the leader's, otherwise it stays for the next round without the lanes already served.  Every round serves at
    // least the leaders, so the loop ends.
    int32_t id = -1;
    for (;;) {
        const unsigned todo = __ballot_sync(act, !bad && id < 0);
        if (todo == 0u) break;
        if (bad || id >= 0) continue;
        const unsigned same = __match_any_sync(todo, fp);
        const int leader = __ffs(same) - 1;
        int32_t got = -1;
        if (lane == leader) got = cc_intern(table, in.hash_mask, fp, q, g, pairs, n_pairs);
        got = __shfl_sync(same, got, leader);
        bool equal = __shfl_sync(same, g, leader) == g;
#pragma unroll
        for (int t = 0; t < 6; ++t) equal &= __shfl_sync(same, q[t], leader) == q[t];
        if (equal) id = got;
    }
    app_pair[i] = bad ? -1 : id;
}

// the pair's class is one of the chunk's
__device__ __forceinline__ bool cc_in_chunk(const CapScratch& s, int32_t cls) {
    return s.a0 < 0 || (cls >= s.a0 && cls - s.a0 < s.K);
}

// the segments a pair visits: class c -> those of buckets [c Z, (c+1) Z), class -1 -> those of class slot G; an affinity
// class a -> those of row a - a0, none outside the chunk
__device__ __forceinline__ void cc_class_segs(const CapScratch& s, int32_t cls, int32_t& first, int32_t& cnt) {
    if (!cc_in_chunk(s, cls)) { first = 0; cnt = 0; return; }
    if (s.a0 >= 0) cls -= s.a0;
    else if (cls < 0) cls = s.G;
    first = s.seg_off[cls * s.Z];
    cnt = s.seg_off[(cls + 1) * s.Z] - first;
}

struct CapPairOut {
    unsigned long long* T;          // [pair] sum of min(cap(n|0), C) over the class
    long long* M;                   // [pair] max of min(cap(d|drv), C) - min(cap(d|0), C), kCapNone = no driver fits
    long long* zone_best;           // [pair] max over zones of T_z + M_z, kCapNone = none
};

__global__ void __launch_bounds__(1024) gp_cc_pair_scan(CapScratch s, const CapPair* __restrict__ pairs, const int32_t* __restrict__ n_pairs,
                                                        long long* __restrict__ pref, CapPairOut out) {
    __shared__ long long sh[33];
    const int32_t np = *n_pairs;
    long long base = 0;
    for (int32_t p0 = 0; p0 < np; p0 += 1024) {
        const int32_t p = p0 + (int32_t)threadIdx.x;
        int32_t first = 0, cnt = 0;
        if (p < np && cc_in_chunk(s, pairs[p].cls)) {
            cc_class_segs(s, pairs[p].cls, first, cnt);
            out.T[p] = 0ull; out.M[p] = kCapNone; out.zone_best[p] = kCapNone;
        }
        long long tot;
        const long long e = cta_excl_scan(cnt, sh, &tot);
        if (p < np) pref[p] = base + e;
        base += tot;
    }
    if (threadIdx.x == 0) pref[np] = base;
}

// ---- the node x pair pass, one chunk of pairs [p0, p1) ------------------------------------------------------------
struct CapPassIn {
    CapScratch s;
    const CapPair* pairs;
    const int32_t* n_pairs;
    const long long* pref;
    CapPairOut out;
    CapSlot* slots;                 // [(p - p0) * ms_stride + ms]
    int32_t ms_stride;              // >= the number of multi-segment buckets
    int32_t p0, p1;
};

__global__ void gp_cc_clear(CapPassIn in) {
    const int32_t p1 = min(in.p1, *in.n_pairs);
    const long long n = (long long)max(p1 - in.p0, 0) * in.ms_stride;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
        in.slots[t] = CapSlot{0ull, kCapNone, 0u, 0};
}

// cap(n|r) clamped to C: the general-class exact division of gangpack_kernels.cuh (multiply-high when the shifted numerator
// fits 32 bits, a true division otherwise), every dimension -- a negative one gives 0 whatever the request
__device__ __forceinline__ uint32_t cc_cap(long long c, long long m, long long g, const CapPair& p) {
    return umin3(cap_dim(c, p.div[0], kCapClamp), cap_dim(m, p.div[1], kCapClamp), cap_dim(g, p.div[2], kCapClamp));
}

__global__ void __launch_bounds__(kCapThreads) gp_cc_pass(CapPassIn in) {
    __shared__ unsigned long long s_sum[kCapThreads / 32];
    __shared__ long long s_max[kCapThreads / 32];
    __shared__ int32_t s_pair, s_seg;
    const int32_t p0 = in.p0, p1 = min(in.p1, *in.n_pairs);
    if (p0 >= p1) return;
    const long long w0 = in.pref[p0], w1 = in.pref[p1];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (long long w = w0 + blockIdx.x; w < w1; w += gridDim.x) {
        if (threadIdx.x == 0) {
            int32_t lo = p0, hi = p1 - 1;                // last p with pref[p] <= w (pairs without segments have pref[p] == pref[p+1])
            while (lo < hi) {
                const int32_t mid = (lo + hi + 1) >> 1;
                if (in.pref[mid] <= w) lo = mid; else hi = mid - 1;
            }
            int32_t first, cnt;
            cc_class_segs(in.s, in.pairs[lo].cls, first, cnt);
            s_pair = lo; s_seg = first + (int32_t)(w - in.pref[lo]);
        }
        __syncthreads();
        const int32_t p = s_pair;
        const CapSeg sg = in.s.segs[s_seg];
        const CapPair& pr = in.pairs[p];
        unsigned long long sum = 0ull;
        long long mx = kCapNone;
        for (int32_t t = (int32_t)threadIdx.x; t < sg.len; t += kCapThreads) {
            const int32_t n = sg.first + t;
            const long long c = in.s.sched[0][n], m = in.s.sched[1][n], g = in.s.sched[2][n];
            const uint32_t c0 = cc_cap(c, m, g, pr);
            sum += c0;
            if (!(pr.drv[0] > c) && !(pr.drv[1] > m) && !(pr.drv[2] > g))       // !driver.GreaterThan(available)
                mx = max(mx, (long long)cc_cap(c - pr.drv[0], m - pr.drv[1], g - pr.drv[2], pr) - (long long)c0);
        }
        sum = warp_sum64(sum);
        mx = warp_max64(mx);
        if (lane == 0) { s_sum[wid] = sum; s_max[wid] = mx; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int k = 1; k < kCapThreads / 32; ++k) { sum += s_sum[k]; mx = max(mx, s_max[k]); }
            atomicAdd(in.out.T + p, sum);
            if (mx != kCapNone) atomicMax(in.out.M + p, mx);
            long long tz = (long long)sum, mz = mx;
            bool complete = sg.ms < 0;                   // the bucket's only segment: T_z, M_z are these
            if (!complete) {                             // the last of the bucket's segments to arrive combines them
                CapSlot* sl = in.slots + (long long)(p - p0) * in.ms_stride + sg.ms;
                atomicAdd(&sl->sum, sum);
                if (mx != kCapNone) atomicMax(&sl->mx, mx);
                __threadfence();
                if (atomicAdd(&sl->arrived, 1u) == (unsigned)(sg.nseg - 1)) {
                    __threadfence();
                    tz = (long long)atomicAdd(&sl->sum, 0ull);
                    mz = atomicMax(&sl->mx, kCapNone);
                    complete = true;
                }
            }
            if (complete && mz != kCapNone) atomicMax(in.out.zone_best + p, tz + mz);
        }
        __syncthreads();                                 // s_pair / s_seg / s_sum are rewritten by the next item
    }
}

// ---- decisions ----------------------------------------------------------------------------------------------------
// packer: 0 tightly-pack, 1 distribute-evenly, 2 az-aware-tightly-pack, 3 single-az-tightly-pack,
// 4 single-az-minimal-fragmentation (gp_binpacker)
__global__ void gp_cc_decide(int32_t n, const int32_t* __restrict__ count, const int32_t* __restrict__ app_pair, const CapPair* __restrict__ pairs,
                             CapPairOut out, int32_t packer, uint8_t* __restrict__ exceeds) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t p = app_pair[i];
    if (p < 0) { exceeds[i] = 1; return; }              // invalid driver: the call fails anyway
    const long long k = count[i];
    bool has;
    if (packer < 3) {
        has = out.M[p] != kCapNone && (long long)out.T[p] + out.M[p] >= k;
    } else {
        // chooseBestResult keeps a zone only with AvgPackingEfficiency.Max > 0: under zero usage some entry of
        // [driver] + ExecutorNodes must reserve a positive amount (minimal fragmentation reserves the driver only)
        const CapPair& pr = pairs[p];
        const bool drv_nz = pr.drv[0] != 0 || pr.drv[1] != 0 || pr.drv[2] != 0;
        const bool exe_nz = pr.div[0].e != 0 || pr.div[1].e != 0 || pr.div[2].e != 0;
        const bool positive = packer == 3 ? (drv_nz || (k >= 1 && exe_nz)) : drv_nz;
        has = positive && out.zone_best[p] >= k;         // kCapNone < 0 <= k
    }
    exceeds[i] = has ? 0 : 1;
}

}  // namespace gp

// gangpack_efficiency.cuh -- the Predicate's cluster-wide packing efficiency on the device, exactly summed.
//
// Reference (EXT = internal/extender, LIB = vendor/github.com/palantir/k8s-spark-scheduler-lib/pkg):
//   computeAvgPackingEfficiencyForResult                  EXT/resource.go:329, 372-381
//   ComputePackingEfficiencies / computePackingEfficiency  LIB/binpack/efficiency.go:66-102 (EVERY node of the metadata)
//   ComputeAvgPackingEfficiency                            LIB/binpack/efficiency.go:114-156
//   SparkBinPack's `reserved` map                          LIB/binpack/binpack.go:72-77 (+ pack_tightly.go:50)
//
// The per-node terms are node_efficiency_values (gangpack_zones.cuh), bit for bit.  Their SUM is not the Go loop's: Go
// iterates a map, whose order is random per call, so the reference's last bits are not reproducible even against itself.
// Here each of the four sums is rounded ONCE, to nearest-even, from its exact real value (what math.fsum returns), which
// is deterministic, independent of the node-table order and within the recursive-summation error bound of every order the
// reference can take.
//
// Exact accumulator: a 256-bit two's-complement fixed-point integer with its least significant bit at 2^-113.
//   Range of a term.  u = sched - avail + reserved is an int64 with |u| < 2^63 (|sched|, |avail| < 2^61 by the snapshot's
//   domain, the add-back and `reserved` < 2^61 by the entry's checks), and every denominator is a non-zero integer with
//   |d| <= 2^61 - 1 (normalizeResource maps 0 to 1).  So |term| <= 2^63 (double(u) may round up to 2^63) and a non-zero
//   |term| > 1 / (2^61 - 1) > 2^-61, i.e. it rounds to at least 2^-61.  A double m * 2^e with a 53-bit m and |value| in
//   [2^-61, 2^63] has e in [-113, 11]: every term is an integer multiple of 2^-113 below 2^(63+113) = 2^176 units.
//   Range of a sum.  < 2^31 nodes, and a row adds at most 2 (k + 1) more terms (new minus old per touched node): every
//   partial sum stays below 2^33 * 2^176 = 2^209 units in magnitude, far inside the 2^255 of the signed 256-bit range.
//   The conversion checks the exponent anyway (kEffErrRange) instead of trusting the bound silently.
// Integer addition is associative, so the warp / block / grid reduction gives the same bits in any order and no
// floating-point atomic is involved.
//
// Base pass: gp_eff_base sums the unreserved terms (reserved = 0) of every node, grid-stride, into one partial per CTA;
// gp_eff_finish adds the partials.  Row pass: gp_eff_rows, one warp per placed row, takes the distinct nodes of
// [driver] + ExecutorNodes (first-occurrence election as in the FIFO kernels, so node-major and round-major lists alike),
// swaps each such node's unreserved terms for its reserved ones in the exact accumulator and rounds once: O(k) per row
// after one O(N) pass per call.
// Segmented (gp_packing_efficiency_groups): the nodes are bucketed by instance group in CSR (seg_off / nodes), n_part CTAs
// of the base pass per segment, gp_eff_finish reduces each segment's partials in a CTA of its own, and a row reads its
// instance group's base and node count.  The whole table is the one-segment case (nodes and seg_off NULL); the sums are
// exact, so the split does not change a bit.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "gangpack_kernels.cuh"
#include "gangpack_zones.cuh"

namespace gp {

constexpr int kEffThreads = 256;
constexpr int kEffFracBits = 113;             // LSB of the fixed point = 2^-113
constexpr int kEffErrRange = 1;               // a term that is no multiple of 2^-113 or reaches 2^79: impossible by the bound above
constexpr int kEffErrQuantity = 2;            // a per-node reserved or added-back amount >= 2^61

struct Fx256 { unsigned long long w[4]; };    // two's complement, w[0] least significant

__device__ __forceinline__ void fx_zero(Fx256& a) { a.w[0] = a.w[1] = a.w[2] = a.w[3] = 0ull; }

__device__ __forceinline__ void fx_add(Fx256& a, const Fx256& b) {
    unsigned long long carry = 0ull;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const unsigned long long s = a.w[i] + b.w[i];
        const unsigned long long c1 = s < a.w[i] ? 1ull : 0ull;
        const unsigned long long t = s + carry;
        const unsigned long long c2 = t < s ? 1ull : 0ull;
        a.w[i] = t;
        carry = c1 | c2;
    }
}

__device__ __forceinline__ void fx_neg(Fx256& a) {
    unsigned long long carry = 1ull;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const unsigned long long t = ~a.w[i] + carry;
        carry = (carry && t == 0ull) ? 1ull : 0ull;
        a.w[i] = t;
    }
}

// a += x exactly; false (a unchanged) if x is not a multiple of 2^-113 or |x| >= 2^79, i.e. its top bit would pass bit 191
// of the accumulator (the bound rules both out)
__device__ __forceinline__ bool fx_add_double(Fx256& a, double x) {
    if (x == 0.0) return true;                                   // +0.0 and -0.0 add nothing
    const unsigned long long bits = (unsigned long long)__double_as_longlong(x);
    const int ex = (int)((bits >> 52) & 0x7ff);
    unsigned long long m = bits & ((1ull << 52) - 1);
    int e;
    if (ex == 0) e = -1074; else { m |= 1ull << 52; e = ex - 1075; }
    int s = e + kEffFracBits;
    if (s < 0) {                                                 // trailing zero bits below 2^-113 may be dropped, nothing else
        if (s <= -53 || (m & ((1ull << -s) - 1)) != 0ull) return false;
        m >>= -s;
        s = 0;
    }
    if (s > 192 - 53) return false;
    // s <= 139: the 53 bits start in limb li = s / 64 (0, 1 or 2) and end in limb li or li + 1, at most bit 191 -- below the
    // sign bit (selects instead of an indexed store keep v in registers)
    const int li = s >> 6, off = s & 63;
    const unsigned long long lo = m << off, hi = off != 0 ? m >> (64 - off) : 0ull;
    Fx256 v;
    v.w[0] = li == 0 ? lo : 0ull;
    v.w[1] = li == 0 ? hi : li == 1 ? lo : 0ull;
    v.w[2] = li == 1 ? hi : li == 2 ? lo : 0ull;
    v.w[3] = li == 2 ? hi : 0ull;
    if (bits >> 63) fx_neg(v);
    fx_add(a, v);
    return true;
}

// limb i of a (selects, not an indexed load: a stays in registers)
__device__ __forceinline__ unsigned long long fx_limb(const Fx256& a, int i) {
    return i == 0 ? a.w[0] : i == 1 ? a.w[1] : i == 2 ? a.w[2] : i == 3 ? a.w[3] : 0ull;
}

// any bit below position p (0 < p <= 256) set?
__device__ __forceinline__ bool fx_any_below(const Fx256& a, int p) {
    bool any = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = p - 64 * i;             // bits of limb i below p
        const unsigned long long mask = r >= 64 ? ~0ull : r > 0 ? (1ull << r) - 1 : 0ull;
        any = any || (a.w[i] & mask) != 0ull;
    }
    return any;
}

// the 64 bits of a from position p upwards (0 <= p < 256)
__device__ __forceinline__ unsigned long long fx_bits_at(const Fx256& a, int p) {
    const int li = p >> 6, off = p & 63;
    unsigned long long v = fx_limb(a, li) >> off;
    if (off != 0) v |= fx_limb(a, li + 1) << (64 - off);
    return v;
}

// round-to-nearest-even of a * 2^-113 to double; zero is +0.0
__device__ __forceinline__ double fx_to_double(Fx256 a) {
    const bool neg = (long long)a.w[3] < 0;
    if (neg) fx_neg(a);
    const int top = a.w[3] ? 3 : a.w[2] ? 2 : a.w[1] ? 1 : a.w[0] ? 0 : -1;
    if (top < 0) return 0.0;
    const int h = 64 * top + 63 - __clzll((long long)fx_limb(a, top));   // highest set bit
    double r;
    if (h <= 52) {
        r = ldexp((double)a.w[0], -kEffFracBits);                  // 53 bits or fewer: exact
    } else {
        int shift = h - 52;
        unsigned long long m = fx_bits_at(a, shift) & ((1ull << 53) - 1);
        const bool half = (fx_bits_at(a, shift - 1) & 1ull) != 0ull;
        const bool sticky = fx_any_below(a, shift - 1);
        if (half && (sticky || (m & 1ull))) {
            ++m;
            if (m == (1ull << 53)) { m >>= 1; ++shift; }
        }
        r = ldexp((double)m, shift - kEffFracBits);
    }
    return neg ? -r : r;
}

__device__ __forceinline__ Fx256 fx_shfl_down(const Fx256& a, int d) {
    Fx256 o;
#pragma unroll
    for (int i = 0; i < 4; ++i) o.w[i] = __shfl_down_sync(0xffffffffu, a.w[i], d);
    return o;
}

// the four sums {cpu, mem, gpu, max} and the number of nodes whose schedulable GPU is non-zero
struct EffAcc {
    Fx256 s[4];
    long long gpu_nodes;
};

__device__ __forceinline__ void acc_zero(EffAcc& a) {
#pragma unroll
    for (int j = 0; j < 4; ++j) fx_zero(a.s[j]);
    a.gpu_nodes = 0;
}
__device__ __forceinline__ void acc_add(EffAcc& a, const EffAcc& b) {
#pragma unroll
    for (int j = 0; j < 4; ++j) fx_add(a.s[j], b.s[j]);
    a.gpu_nodes += b.gpu_nodes;
}
// lane 0 ends with the warp's sum
__device__ __forceinline__ void acc_warp_reduce(EffAcc& a) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        EffAcc o;
#pragma unroll
        for (int j = 0; j < 4; ++j) o.s[j] = fx_shfl_down(a.s[j], d);
        o.gpu_nodes = __shfl_down_sync(0xffffffffu, a.gpu_nodes, d);
        acc_add(a, o);
    }
}
// thread 0 ends with the CTA's sum (blockDim.x == kEffThreads)
__device__ __forceinline__ void acc_block_reduce(EffAcc& a) {
    __shared__ EffAcc part[kEffThreads / 32];
    acc_warp_reduce(a);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) part[warp] = a;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < kEffThreads / 32; ++w) acc_add(a, part[w]);
}

// AvailableResources of a node where the snapshot holds them now: its slot when it is in an order (FIFO, reservations and
// usage deltas charge the slots), the node-table copy otherwise.  Read-only.
struct SnapshotAvail {
    const longlong2* pair;
    const long long* sgpu;
    const int32_t* node_slot;
    const long long* ncpu;
    const long long* nmem;
    const long long* ngpu;
    __device__ __forceinline__ void load(int32_t n, long long& c, long long& m, long long& g) const {
        const int32_t sl = node_slot[n];
        if (sl >= 0) { const longlong2 v = pair[sl]; c = v.x; m = v.y; g = sgpu[sl]; }
        else { c = ncpu[n]; m = nmem[n]; g = ngpu[n]; }
    }
};

// a += the four terms of node n with (avail + back) available and `res` reserved, each multiplied by sign (+1 / -1)
__device__ __forceinline__ bool acc_node_terms(EffAcc& a, const long long* const* sched, const long long* av, const long long* back,
                                               const long long* res, double sign) {
    double c, m, g;
    bool hg;
    const double mx = node_efficiency_values(sched[0][0], sched[1][0], sched[2][0], av[0] + back[0], av[1] + back[1], av[2] + back[2],
                                             res[0], res[1], res[2], c, m, g, hg);
    bool ok = fx_add_double(a.s[0], sign * c) && fx_add_double(a.s[1], sign * m) && fx_add_double(a.s[3], sign * mx);
    if (hg) ok = ok && fx_add_double(a.s[2], sign * g);
    return ok;
}

struct EffBaseIn {
    SnapshotAvail av;
    const long long* sched[3];       // SchedulableResources [3][n_nodes]
    int32_t n_nodes;
    const int32_t* nodes;            // segmented: the nodes bucketed by segment, or NULL (every node, one segment)
    const int32_t* seg_off;          // segmented: [segments + 1] CSR of nodes, or NULL
    int32_t n_part;                  // CTAs per segment (the grid is segments x n_part)
};

// unreserved terms of every node of segment blockIdx.x / n_part -> partial[blockIdx.x]
__global__ void __launch_bounds__(kEffThreads) gp_eff_base(EffBaseIn in, EffAcc* __restrict__ partial, int* __restrict__ err) {
    EffAcc a;
    acc_zero(a);
    bool ok = true;
    const long long zero[3] = {0, 0, 0};
    const int32_t sg = blockIdx.x / in.n_part, part = blockIdx.x - sg * in.n_part;
    const int32_t lo = in.seg_off ? in.seg_off[sg] : 0, hi = in.seg_off ? in.seg_off[sg + 1] : in.n_nodes;
    for (int32_t t = lo + part * kEffThreads + threadIdx.x; t < hi; t += in.n_part * kEffThreads) {
        const int32_t n = in.nodes ? in.nodes[t] : t;
        long long av[3];
        in.av.load(n, av[0], av[1], av[2]);
        const long long* sc[3] = {in.sched[0] + n, in.sched[1] + n, in.sched[2] + n};
        ok = acc_node_terms(a, sc, av, zero, zero, 1.0) && ok;
        a.gpu_nodes += sc[2][0] != 0 ? 1 : 0;
    }
    if (!ok) atomicOr(err, kEffErrRange);
    acc_block_reduce(a);
    if (threadIdx.x == 0) partial[blockIdx.x] = a;
}

// one CTA per segment: partial[blockIdx.x * n_partial ..][0 .. n_partial) -> base[blockIdx.x]
__global__ void __launch_bounds__(kEffThreads) gp_eff_finish(const EffAcc* __restrict__ partial, int32_t n_partial, EffAcc* __restrict__ base) {
    EffAcc a;
    acc_zero(a);
    partial += (size_t)blockIdx.x * n_partial;
    for (int32_t i = threadIdx.x; i < n_partial; i += kEffThreads) acc_add(a, partial[i]);
    acc_block_reduce(a);
    if (threadIdx.x == 0) base[blockIdx.x] = a;
}

struct EffRowsIn {
    SnapshotAvail av;
    const long long* sched[3];
    SixCols cols;                     // drv cpu, mem, gpu, exe cpu, mem, gpu (gpu columns may be NULL = 0)
    const int32_t* count;
    const int64_t* off;               // ExecutorNodes offsets
    const int32_t* driver;
    const int32_t* exec;
    const EffAcc* base;               // [segments]
    const int32_t* group;             // segmented: each row's segment (instance group), or NULL (segment 0)
    const int32_t* seg_off;           // segmented: [segments + 1], a segment's node count is its length; NULL: n_nodes
    int32_t n_apps;
    int32_t n_nodes;
    int32_t executors_reserved;       // 0: minimal-fragmentation (the driver alone is in `reserved`)
    int32_t charged;                  // gp_mode: 0 nothing to add back; 1 sparkResourceUsage's map; 2 every pod
};

// v = a + cnt * e in [0, 2^61)?  (a in [0, 2^61), e >= 0, cnt >= 0)
__device__ __forceinline__ bool amount_fits(long long a, long long cnt, long long e, long long& v) {
    if (cnt != 0 && e > (kMaxQuantity - 1 - a) / cnt) return false;
    v = a + cnt * e;
    return true;
}

__global__ void __launch_bounds__(kEffThreads) gp_eff_rows(EffRowsIn in, double* __restrict__ avg_out, int* __restrict__ err) {
    const int lane = threadIdx.x & 31;
    const int32_t i = (int32_t)((blockIdx.x * (unsigned)kEffThreads + threadIdx.x) >> 5);
    if (i >= in.n_apps) return;
    const int32_t d = in.driver[i];
    if (d < 0) {                                                   // no placement: WorstAvgPackingEfficiency
        if (lane < 4) avg_out[4 * (int64_t)i + lane] = 0.0;
        return;
    }
    const int32_t k = in.count[i] > 0 ? in.count[i] : 0;
    const int32_t* ex = in.exec + in.off[i];
    const long long drv[3] = {in.cols.p[0][i], in.cols.p[1][i], in.cols.p[2] ? in.cols.p[2][i] : 0};
    const long long exe[3] = {in.cols.p[3][i], in.cols.p[4][i], in.cols.p[5] ? in.cols.p[5][i] : 0};
    EffAcc delta;
    acc_zero(delta);
    bool ok = true, fits = true;
    // node n with isd (it hosts the driver) and cnt executors of this placement: unreserved terms out, reserved terms in
    auto swap_node = [&](int32_t n, long long isd, long long cnt) {
        long long res[3], back[3], av[3];
        const long long zero[3] = {0, 0, 0};
        for (int r = 0; r < 3; ++r) {
            fits = amount_fits(isd * drv[r], in.executors_reserved ? cnt : 0, exe[r], res[r]) && fits;
            if (in.charged == 2) fits = amount_fits(isd * drv[r], cnt, exe[r], back[r]) && fits;
            else if (in.charged == 1) back[r] = cnt > 0 ? exe[r] : isd * drv[r];      // sparkpods.go:139-146
            else back[r] = 0;
        }
        if (!fits) return;
        in.av.load(n, av[0], av[1], av[2]);
        const long long* sc[3] = {in.sched[0] + n, in.sched[1] + n, in.sched[2] + n};
        ok = acc_node_terms(delta, sc, av, zero, zero, -1.0) && ok;
        ok = acc_node_terms(delta, sc, av, back, res, 1.0) && ok;
    };
    bool hosts = false;                                            // the driver's node is among ExecutorNodes
    for (int32_t t = lane; t < k; t += 32) {
        const int32_t n = ex[t];
        hosts = hosts || n == d;
        // one lane per distinct node: the first entry that names it, with the number of entries that do
        bool first = t == 0 || ex[t - 1] != n;
        for (int32_t u = 0; first && u + 1 < t; ++u) first = ex[u] != n;
        if (first) {
            long long cnt = 0;
            for (int32_t u = t; u < k; ++u) cnt += ex[u] == n ? 1 : 0;
            swap_node(n, n == d ? 1 : 0, cnt);
        }
    }
    hosts = __any_sync(0xffffffffu, hosts);
    if (lane == 0 && !hosts) swap_node(d, 1, 0);
    if (__any_sync(0xffffffffu, !fits)) { if (lane == 0) atomicOr(err, kEffErrQuantity); return; }
    if (!ok) atomicOr(err, kEffErrRange);
    acc_warp_reduce(delta);
    if (lane == 0) {
        const int32_t g = in.group ? in.group[i] : 0;
        EffAcc t = in.base[g];
        acc_add(t, delta);
        const double length = fmax((double)(in.seg_off ? in.seg_off[g + 1] - in.seg_off[g] : in.n_nodes), 1.0);
        double* o = avg_out + 4 * (int64_t)i;
        o[0] = fx_to_double(t.s[0]) / length;
        o[1] = fx_to_double(t.s[1]) / length;
        o[2] = t.gpu_nodes == 0 ? 1.0 : fx_to_double(t.s[2]) / (double)t.gpu_nodes;
        o[3] = fx_to_double(t.s[3]) / length;
    }
}

}  // namespace gp

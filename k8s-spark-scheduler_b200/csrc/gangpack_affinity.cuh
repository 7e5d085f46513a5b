// gangpack_affinity.cuh -- a driver's required node affinity matched against every node on the device.
//
// Reference (K8S = vendor/k8s.io):
//   GetRequiredNodeAffinity / RequiredNodeAffinity.Match      K8S/component-helpers/scheduling/corev1/nodeaffinity/nodeaffinity.go:297-324
//   LazyErrorNodeSelector.Match, nodeSelectorTerm.match       nodeaffinity.go:56-103, 152-201
//   Requirement.Matches                                       K8S/apimachinery/pkg/labels/selector.go:218-262
// used by selectDriverNode (EXT/resource.go:292-298) and DoesPodExceedClusterCapacity (EXT/unschedulablepods.go:133-139)
// through utils.ListWithPredicate.
//
// Strings never reach the device: label keys and values are interned ids, a node's labels are sorted by key id, each
// requirement's value set is a sorted list of value ids, and whatever needs the strings (NewRequirement's validation, ParseInt
// of a node's label value, metadata.name -> node index) the caller has already done.  One outcome per (affinity, node):
//   1. nodeSelector: every (key, value) present and equal, else no match -- whatever the terms would have said;
//   2. no required affinity: match;
//   3. terms in order: a term flagged with a parse error records an error and is skipped, a term without requirements is
//      skipped, a term matches when all its requirements do, and the first matching term is a match;
//   4. otherwise no match, an error if some term recorded one.
//
// The labels come from one of two sources, a template parameter of aff_req / aff_outcome / gp_aff_match:
//   AffLabelsIn        the per-call CSR of gp_node_labels, ParseInt per label entry;
//   AffLabelsResident  the label table's fixed-stride rows (gangpack_label_table.cu), read through the call's node_id (-1: no
//                      labels), ParseInt per value id.
// Both give a node's labels as a range [lo, hi) of one key column and one value column, so the program runs unchanged.
//
// Kernel gp_aff_labels: thread per node, checks its per-call labels (ids in range, keys strictly ascending) -- once per call,
// whatever the number of affinities.  The resident rows were checked when they were written; gp_aff_ids checks the call's
// node ids against the table instead.
// Kernel gp_aff_match: grid (node tiles, affinity).  The CTA stages its affinity's program in shared memory (or reads it
// from global memory when it is larger than kAffSmem bytes); each thread runs the program on one node, finding each key by
// binary search in the node's labels and each In / NotIn value by binary search in the requirement's values.  Bitmap words
// come from __ballot_sync, n_match / n_error from one atomic per warp.  Work per (affinity, node): O(requirements x log labels).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "gangpack_kernels.cuh"
#include "gangpack_labels.cuh"

namespace gp {

constexpr int kAffThreads = 256;
constexpr int kAffSmem = 16 * 1024;       // bytes of shared memory for one affinity's program

enum : int32_t {                          // gp_aff_op
    kAffIn = 0, kAffNotIn = 1, kAffExists = 2, kAffDoesNotExist = 3, kAffGt = 4, kAffLt = 5,
    kAffFieldNameIn = 6, kAffFieldNameNotIn = 7,
};

enum : int {
    kAffErrLabelKey = 1,                  // a node's label key out of range, or keys not strictly ascending
    kAffErrLabelVal = 2,                  // a node's label value out of range
};

enum : int {
    kAffErrNodeId = 4,                    // a resident node id outside [-1, n_node_ids)
};

struct AffLabelsIn {
    int32_t n, n_keys, n_values;
    const long long* off;                 // [n + 1]
    const int32_t* key;
    const int32_t* val;
    const uint8_t* int_ok;                // NULL: no value parses
    const long long* ival;
    __device__ __forceinline__ void range(int32_t node, long long& lo, long long& hi) const { lo = off[node]; hi = off[node + 1]; }
    __device__ __forceinline__ bool int_at(long long e, long long& v) const {
        if (!int_ok || !int_ok[e]) return false;
        v = ival[e];
        return true;
    }
};

struct AffProgIn {
    int32_t n_aff;
    const long long* sel_off;             // [n_aff + 1]
    const int32_t* sel_key;
    const int32_t* sel_val;
    const uint8_t* has_required;          // [n_aff]
    const long long* term_off;            // [n_aff + 1]
    const long long* term_req_off;        // [n_terms + 1]
    const uint8_t* term_err;              // [n_terms]
    const int32_t* req_op;
    const int32_t* req_key;
    const long long* req_int;             // Gt / Lt bound; metadata.name: node index or -1
    const long long* req_val_off;         // [n_req + 1]
    const int32_t* req_val;
};

struct AffOut {
    uint32_t* member;                     // [rows][words]: affinity a in row a - row0
    int32_t* n_match;                     // [n_aff]
    int32_t* n_error;                     // [n_aff]
    int32_t words;
    int32_t row0;
};

// One affinity's program: every pointer is rebased so that index 0 is the affinity's first element, offsets stay absolute
// (subtract the *_base to index)
struct AffView {
    const int32_t* sel_key; const int32_t* sel_val; int32_t n_sel;
    const long long* term_req_off; const uint8_t* term_err; int32_t n_terms;
    const int32_t* req_op; const int32_t* req_key; const long long* req_int; const long long* req_val_off; long long req_base;
    const int32_t* req_val; long long val_base;
    bool has_required;
};

template <class Lab>
__device__ __forceinline__ bool aff_req(const AffView& p, long long r, const Lab& L, long long lo, long long hi, int32_t node) {
    const int32_t op = p.req_op[r];
    if (op == kAffFieldNameIn) return (long long)node == p.req_int[r];
    if (op == kAffFieldNameNotIn) return (long long)node != p.req_int[r];
    const long long at = aff_find(L.key, lo, hi, p.req_key[r]);
    switch (op) {
    case kAffIn:
    case kAffNotIn: {
        if (at < 0) return op == kAffNotIn;
        const bool has = aff_find(p.req_val, p.req_val_off[r] - p.val_base, p.req_val_off[r + 1] - p.val_base, L.val[at]) >= 0;
        return op == kAffIn ? has : !has;
    }
    case kAffExists: return at >= 0;
    case kAffDoesNotExist: return at < 0;
    case kAffGt:
    case kAffLt: {
        long long v;
        if (at < 0 || !L.int_at(at, v)) return false;                    // ParseInt failed: no match, not an error
        return op == kAffGt ? v > p.req_int[r] : v < p.req_int[r];
    }
    default: return false;
    }
}

// 0 no match, 1 match, 2 error
template <class Lab>
__device__ __forceinline__ int aff_outcome(const AffView& p, const Lab& L, int32_t node) {
    long long lo, hi;
    L.range(node, lo, hi);
    for (int32_t t = 0; t < p.n_sel; ++t) {
        const long long at = aff_find(L.key, lo, hi, p.sel_key[t]);
        if (at < 0 || L.val[at] != p.sel_val[t]) return 0;
    }
    if (!p.has_required) return 1;
    bool errored = false;
    for (int32_t t = 0; t < p.n_terms; ++t) {
        if (p.term_err[t]) { errored = true; continue; }
        const long long r0 = p.term_req_off[t] - p.req_base, r1 = p.term_req_off[t + 1] - p.req_base;
        if (r0 == r1) continue;                                          // an empty term selects nothing
        bool all = true;
        for (long long r = r0; r < r1 && all; ++r) all = aff_req(p, r, L, lo, hi, node);
        if (all) return 1;
    }
    return errored ? 2 : 0;
}

template <typename T>
__device__ __forceinline__ T* aff_stage(unsigned char*& at, const T* src, long long n) {
    T* dst = reinterpret_cast<T*>(at);
    for (long long i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
    at += ((size_t)n * sizeof(T) + 7) & ~(size_t)7;
    return dst;
}

__global__ void gp_aff_labels(AffLabelsIn L, int* err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L.n) return;
    const long long lo = L.off[i], hi = L.off[i + 1];
    int bad = 0;
    for (long long e = lo; e < hi; ++e) {
        const int32_t k = L.key[e], v = L.val[e];
        if (k < 0 || k >= L.n_keys || (e > lo && k <= L.key[e - 1])) bad |= kAffErrLabelKey;
        if (v < 0 || v >= L.n_values) bad |= kAffErrLabelVal;
    }
    if (bad) atomicOr(err, bad);
}

// thread per node of a resident call: its label-table id in [-1, n_rows)
__global__ void gp_aff_ids(AffLabelsResident L, int* err) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L.n) return;
    const int32_t r = L.node_id[i];
    if (r < -1 || r >= L.n_rows) atomicOr(err, kAffErrNodeId);
}

// affinities a_base + blockIdx.y (gridDim.y <= 65535: more affinities take more launches)
template <class Lab>
__global__ void __launch_bounds__(kAffThreads) gp_aff_match(Lab L, AffProgIn P, AffOut out, int32_t a_base) {
    __shared__ __align__(16) unsigned char s_prog[kAffSmem];
    const int32_t a = a_base + (int32_t)blockIdx.y;
    const long long s0 = P.sel_off[a], s1 = P.sel_off[a + 1], t0 = P.term_off[a], t1 = P.term_off[a + 1];
    const long long r0 = P.term_req_off[t0], r1 = P.term_req_off[t1];
    const long long v0 = P.req_val_off[r0], v1 = P.req_val_off[r1];
    const long long ns = s1 - s0, nt = t1 - t0, nr = r1 - r0, nv = v1 - v0;
    AffView p;
    p.n_sel = (int32_t)ns; p.n_terms = (int32_t)nt; p.req_base = r0; p.val_base = v0;
    p.has_required = P.has_required[a] != 0;
    auto r8 = [](long long b) { return (b + 7) & ~7LL; };                // aff_stage's footprint of each piece
    const long long bytes = 8 * (nt + 1) + 8 * nr + 8 * (nr + 1) + 2 * r8(4 * ns) + 2 * r8(4 * nr) + r8(4 * nv) + r8(nt);
    if (bytes <= kAffSmem) {
        unsigned char* at = s_prog;
        p.term_req_off = aff_stage(at, P.term_req_off + t0, nt + 1);
        p.req_int = aff_stage(at, P.req_int + r0, nr);
        p.req_val_off = aff_stage(at, P.req_val_off + r0, nr + 1);
        p.sel_key = aff_stage(at, P.sel_key + s0, ns);
        p.sel_val = aff_stage(at, P.sel_val + s0, ns);
        p.req_op = aff_stage(at, P.req_op + r0, nr);
        p.req_key = aff_stage(at, P.req_key + r0, nr);
        p.req_val = aff_stage(at, P.req_val + v0, nv);
        p.term_err = aff_stage(at, P.term_err + t0, nt);
        __syncthreads();
    } else {                                                             // too large for shared memory: read it in place
        p.term_req_off = P.term_req_off + t0; p.req_int = P.req_int + r0; p.req_val_off = P.req_val_off + r0;
        p.sel_key = P.sel_key + s0; p.sel_val = P.sel_val + s0; p.req_op = P.req_op + r0; p.req_key = P.req_key + r0;
        p.req_val = P.req_val + v0; p.term_err = P.term_err + t0;
    }
    const int32_t i = blockIdx.x * kAffThreads + threadIdx.x;
    int outcome = 0;
    if (i < L.n) outcome = aff_outcome(p, L, i);
    const unsigned hit = __ballot_sync(kFull, outcome == 1), miss = __ballot_sync(kFull, outcome == 2);
    const int32_t base = i & ~31;
    if ((threadIdx.x & 31) == 0 && base < L.n) {
        out.member[(long long)(a - out.row0) * out.words + (base >> 5)] = hit;
        if (hit) atomicAdd(out.n_match + a, __popc(hit));
        if (miss) atomicAdd(out.n_error + a, __popc(miss));
    }
}

}  // namespace gp

// gangpack_overhead.cuh -- the overhead computer's per-call side on the device: PodHasReservation for every recorded pod and
// the per-node sums of the pods without one.
//
// Reference (EXT = internal/extender):
//   OverheadComputer.getOverheadByNode / computeNodeOverhead    EXT/overhead.go:105-153
//   PodHasReservation                                          EXT/resourcereservations.go:115-132
//   SoftReservationStore.GetExecutorSoftReservation            internal/cache/softreservations.go:136-152
//
// Strings never reach the device: node names, (namespace, spark-app-id) pairs, spark-app-ids and pod names are dense ids.
//
// Kernel gp_oh_dir: the directories over the id spaces -- app key -> ResourceReservation index, app id -> soft-store index,
// node id -> query row -- each written with atomicCAS, so an id given twice is seen as a duplicate.
// Kernel gp_oh_insert: thread per (reservation, pod name) entry; the entry's reservation comes from a binary search of the
// CSR offsets, and (reservation index, name) packed into 64 bits goes into an open-addressing hash set (linear probing,
// at most half full).  The soft store's entries use indices n_rr + s, so one set serves both.  A membership test is then
// O(1) expected, whatever the number of pods an application reserves.
// Kernel gp_oh_pods: thread per record slot.  Classifies the pod, and adds the requests of a pod without a reservation on a
// listed node into that node's row.  Sums are exact and independent of order: each request (< 2^61) is split into its low
// 32 bits and the rest, each half summed by a 64-bit atomicAdd (fewer than 2^31 slots: neither half-sum wraps).
// Kernel gp_oh_finish: thread per listed node; recombines the halves and flags a sum >= 2^61.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "gangpack_kernels.cuh"

namespace gp {

constexpr int kOhThreads = 256;
constexpr unsigned long long kOhEmpty = ~0ull;        // hash slot never written (the table is memset to 0xff)

enum : int {
    kOhErrRange = 1,            // an id out of its range
    kOhErrDuplicate = 2,        // a query node id, rr_app_key or soft_app_id given twice
    kOhErrAppPair = 4,          // app_key and app_id disagree on -1
    kOhErrNegative = 8,         // a negative request
    kOhErrRequest = 16,         // a request >= 2^61
    kOhErrSum = 32,             // a per-node sum >= 2^61
};

struct OhDirIn {
    int32_t n_rr, n_soft, n_nodes;
    int32_t n_app_keys, n_app_ids, n_node_ids;
    const int32_t* rr_app_key;
    const int32_t* soft_app_id;
    const int32_t* node_ids;
};

struct OhMaps {
    int32_t* rr_of_key;                 // [n_app_keys] ResourceReservation index, -1 = none
    int32_t* soft_of_app;               // [n_app_ids] soft-store index, -1 = none
    int32_t* row_of_node;               // [n_node_ids] query row, -1 = not listed
    unsigned long long* set;            // [mask + 1] (reservation index << 32 | name id), kOhEmpty = free
    uint32_t mask;
    int32_t n_rr;                       // soft-store index s is reservation index n_rr + s in the set
};

struct OhSetIn {
    const long long* rr_off;            // [n_rr + 1]
    const int32_t* rr_name;
    const long long* soft_off;          // [n_soft + 1]
    const int32_t* soft_name;
    int32_t n_rr, n_soft, n_names;
    long long n_rr_entries, n_soft_entries;
};

struct OhPodsIn {
    long long n;
    int32_t n_node_ids, n_app_keys, n_app_ids, n_names;
    const int32_t* node_id;
    const long long* req[3];            // cpu, mem, gpu (gpu may be NULL)
    const uint8_t* listed;              // NULL = all
    const int32_t* app_key;
    const int32_t* app_id;
    const int32_t* name_id;
    const uint8_t* is_executor;         // NULL = none
    const uint8_t* spark_scheduler;     // NULL = none
    uint8_t* has_reservation;           // [n]
};

// acc[(2 * k + half) * n_rows + row]: k = set * 3 + dimension (set 0 overhead, 1 non-schedulable overhead), half 0 = the low
// 32 bits of each request, 1 = the rest
struct OhAcc {
    unsigned long long* acc;
    unsigned long long* n_warned;
    int32_t n_rows;
};

__device__ __forceinline__ uint32_t oh_hash(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return (uint32_t)k;
}

__device__ __forceinline__ unsigned long long oh_key(int32_t reservation, int32_t name) {
    return ((unsigned long long)(uint32_t)reservation << 32) | (uint32_t)name;
}

__device__ __forceinline__ bool oh_member(const OhMaps& M, int32_t reservation, int32_t name) {
    const unsigned long long k = oh_key(reservation, name);
    for (uint32_t h = oh_hash(k) & M.mask;; h = (h + 1) & M.mask) {
        const unsigned long long v = M.set[h];
        if (v == k) return true;
        if (v == kOhEmpty) return false;
    }
}

__global__ void gp_oh_dir(OhDirIn D, OhMaps M, int* err) {
    const long long total = (long long)D.n_rr + D.n_soft + D.n_nodes;
    int bad = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int32_t id, lim, at;
        int32_t* dir;
        if (i < D.n_rr) { at = (int32_t)i; id = D.rr_app_key[at]; lim = D.n_app_keys; dir = M.rr_of_key; }
        else if (i < (long long)D.n_rr + D.n_soft) { at = (int32_t)(i - D.n_rr); id = D.soft_app_id[at]; lim = D.n_app_ids; dir = M.soft_of_app; }
        else { at = (int32_t)(i - D.n_rr - D.n_soft); id = D.node_ids[at]; lim = D.n_node_ids; dir = M.row_of_node; }
        if (id < 0 || id >= lim) { bad |= kOhErrRange; continue; }
        if (atomicCAS(dir + id, -1, at) != -1) bad |= kOhErrDuplicate;
    }
    if (bad) atomicOr(err, bad);
}

__global__ void gp_oh_insert(OhSetIn S, OhMaps M, int* err) {
    const long long total = S.n_rr_entries + S.n_soft_entries;
    int bad = 0;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const bool soft = e >= S.n_rr_entries;
        const long long x = soft ? e - S.n_rr_entries : e;
        const long long* off = soft ? S.soft_off : S.rr_off;
        const int32_t name = soft ? S.soft_name[x] : S.rr_name[x];
        if (name < 0 || name >= S.n_names) { bad |= kOhErrRange; continue; }
        int32_t lo = 0, hi = soft ? S.n_soft : S.n_rr;           // the last r with off[r] <= x (empty segments skipped)
        while (hi - lo > 1) {
            const int32_t mid = (lo + hi) >> 1;
            if (off[mid] <= x) lo = mid; else hi = mid;
        }
        const unsigned long long k = oh_key(soft ? S.n_rr + lo : lo, name);
        for (uint32_t h = oh_hash(k) & M.mask;; h = (h + 1) & M.mask) {
            const unsigned long long prev = atomicCAS(M.set + h, kOhEmpty, k);
            if (prev == kOhEmpty || prev == k) break;               // inserted, or a repeated name of the same reservation
        }
    }
    if (bad) atomicOr(err, bad);
}

__device__ __forceinline__ void oh_add(const OhAcc& A, int k, int32_t row, long long v) {
    if (!v) return;
    atomicAdd(A.acc + (size_t)(2 * k) * A.n_rows + row, (unsigned long long)v & 0xffffffffull);
    if (v >> 32) atomicAdd(A.acc + (size_t)(2 * k + 1) * A.n_rows + row, (unsigned long long)v >> 32);
}

__global__ void __launch_bounds__(kOhThreads) gp_oh_pods(OhPodsIn P, OhMaps M, OhAcc A, int* err) {
    const long long i = (long long)blockIdx.x * kOhThreads + threadIdx.x;
    int bad = 0;
    bool warn = false;
    if (i < P.n) {
        uint8_t has = 0;
        const int32_t node = P.node_id[i];
        if (node != -1) {
            long long q[3];
            for (int d = 0; d < 3; ++d) {
                q[d] = P.req[d] ? P.req[d][i] : 0;
                if (q[d] < 0) bad |= kOhErrNegative;
                else if (q[d] >= kMaxQuantity) bad |= kOhErrRequest;
            }
            if (node < 0 || node >= P.n_node_ids) bad |= kOhErrRange;
            if (!P.listed || P.listed[i]) {
                const int32_t ak = P.app_key[i], ai = P.app_id[i], nm = P.name_id[i];
                if (ak < -1 || ak >= P.n_app_keys || ai < -1 || ai >= P.n_app_ids || nm < 0 || nm >= P.n_names) bad |= kOhErrRange;
                else if ((ak < 0) != (ai < 0)) bad |= kOhErrAppPair;
                bool rr_exists = false;
                if (!bad && ak >= 0) {
                    const int32_t r = M.rr_of_key[ak];
                    rr_exists = r >= 0;
                    if (rr_exists && oh_member(M, r, nm)) has = 1;
                    else if (P.is_executor && P.is_executor[i]) {
                        const int32_t s = M.soft_of_app[ai];
                        if (s >= 0 && oh_member(M, M.n_rr + s, nm)) has = 1;
                    }
                }
                const int32_t row = bad ? -1 : M.row_of_node[node];
                if (!has && row >= 0) {
                    const bool spark = P.spark_scheduler && P.spark_scheduler[i];
                    for (int d = 0; d < 3; ++d) {
                        oh_add(A, d, row, q[d]);
                        if (!spark) oh_add(A, 3 + d, row, q[d]);
                    }
                    warn = spark && rr_exists;
                }
            }
        }
        if (P.has_reservation) P.has_reservation[i] = has;
    }
    const unsigned w = __ballot_sync(kFull, warn);
    if ((threadIdx.x & 31) == 0 && w) atomicAdd(A.n_warned, (unsigned long long)__popc(w));
    if (bad) atomicOr(err, bad);
}

// out[k * n_rows + row], k as in OhAcc
__global__ void gp_oh_finish(OhAcc A, long long* out, int* err) {
    const int32_t row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= A.n_rows) return;
    bool over = false;
    for (int k = 0; k < 6; ++k) {
        const unsigned long long lo = A.acc[(size_t)(2 * k) * A.n_rows + row], hi = A.acc[(size_t)(2 * k + 1) * A.n_rows + row];
        // hi < 2^29 keeps (hi << 32) + lo below 2^61 + 2^63: no wrap before the comparison
        const unsigned long long t = (hi << 32) + lo;
        over |= hi >= (1ull << 29) || t >= (unsigned long long)kMaxQuantity;
        out[(size_t)k * A.n_rows + row] = (long long)t;
    }
    if (over) atomicOr(err, kOhErrSum);
}

}  // namespace gp

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
// Kernel gp_oh_pods<Lookup>: thread per record slot.  Classifies the pod through Lookup (OhCallLookup: the directories and the
// set above; OhTableLookup: the resident table's RR flags and member set), and adds the requests of a pod without a reservation on a
// listed node into that node's row.  Sums are exact and independent of order: each request (< 2^61) is split into its low
// 32 bits and the rest, each half summed by a 64-bit atomicAdd (fewer than 2^31 slots: neither half-sum wraps).
// Kernel gp_oh_finish: thread per listed node; recombines the halves and flags a sum >= 2^61.
//
// The resident table (gp_overhead_table_*, gangpack_overhead_table.cu) keeps the slot columns, one RR flag per app key and a
// member set of 64-bit keys (kind << 62 | app << 31 | name) on the device; a query is gp_oh_dir over the listed nodes alone,
// then gp_oh_pods<OhTableLookup> and gp_oh_finish.  An update runs
//   gp_oht_check    thread per write: every range, request and duplicate check; sets the error word and writes nothing else
//   gp_oht_rehash   (when the set could pass half full) every live key of the old cells into a new, larger set
//   gp_oht_apply    thread per slot write, RR flag write and member removal (present = 0); nothing when the error word is set
//   gp_oht_insert   thread per member insertion (present = 1); nothing when the error word is set
// Removals and insertions are separate launches, and a delta names each key at most once, so every key has one writer.
// Deletion leaves a tombstone; an insertion only ever claims an empty cell, so a probe for a key that is present meets it
// before the first empty cell.  Tombstones count towards the load and are dropped by gp_oht_rehash.
// The kernels are static: gangpack_marker.cu and gangpack_overhead_table.cu each launch their own copy.
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

static __global__ void gp_oh_dir(OhDirIn D, OhMaps M, int* err) {
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

static __global__ void gp_oh_insert(OhSetIn S, OhMaps M, int* err) {
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

// The membership lookup of gp_node_overhead: directories and the per-call set of (reservation index, name)
struct OhCallLookup {
    OhMaps M;
    __device__ int32_t row(int32_t node) const { return M.row_of_node[node]; }
    // PodHasReservation for a labelled pod -> has; *rr_exists: the ResourceReservation (namespace, appID) exists
    __device__ bool has(int32_t ak, int32_t ai, int32_t nm, bool exe, bool* rr_exists) const {
        const int32_t r = M.rr_of_key[ak];
        *rr_exists = r >= 0;
        if (*rr_exists && oh_member(M, r, nm)) return true;
        if (!exe) return false;
        const int32_t s = M.soft_of_app[ai];
        return s >= 0 && oh_member(M, M.n_rr + s, nm);
    }
};

template <class Lookup>
__global__ void __launch_bounds__(kOhThreads) gp_oh_pods(OhPodsIn P, Lookup L, OhAcc A, int* err) {
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
                if (!bad && ak >= 0 && L.has(ak, ai, nm, P.is_executor && P.is_executor[i], &rr_exists)) has = 1;
                const int32_t row = bad ? -1 : L.row(node);
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
static __global__ void gp_oh_finish(OhAcc A, long long* out, int* err) {
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

// ---- the resident table -------------------------------------------------------------------------------------------------
constexpr unsigned long long kOhTomb = ~0ull - 1;     // a removed member; bit 63 is clear in every real key

enum : int {
    kOhtErrRange = 1,           // a slot, id or member kind out of its range
    kOhtErrDuplicate = 2,       // a slot, rr_app_key or member triple given twice in one delta
    kOhtErrAppPair = 4,         // app_key and app_id disagree on -1
    kOhtErrNegative = 8,        // a negative request
    kOhtErrRequest = 16,        // a request >= 2^61
};

__device__ __forceinline__ unsigned long long oht_key(int kind, int32_t app, int32_t name) {
    return ((unsigned long long)kind << 62) | ((unsigned long long)(uint32_t)app << 31) | (uint32_t)name;
}

struct OhtSet {
    unsigned long long* cell;           // [mask + 1] keys, kOhEmpty or kOhTomb
    uint32_t mask;
};

__device__ __forceinline__ bool oht_find(const OhtSet& S, unsigned long long k, uint32_t* at) {
    for (uint32_t h = oh_hash(k) & S.mask;; h = (h + 1) & S.mask) {
        const unsigned long long v = S.cell[h];
        if (v == k) { *at = h; return true; }
        if (v == kOhEmpty) return false;
    }
}

// k into the first empty cell of its probe sequence (k is absent and no other thread inserts k)
__device__ __forceinline__ void oht_claim(const OhtSet& S, unsigned long long k) {
    for (uint32_t h = oh_hash(k) & S.mask;; h = (h + 1) & S.mask)
        if (S.cell[h] == kOhEmpty && atomicCAS(S.cell + h, kOhEmpty, k) == kOhEmpty) return;
}

// The table's device columns, as gp_oh_pods reads them and gp_oht_apply writes them
struct OhtCols {
    int32_t* node_id;
    long long* req[3];
    uint8_t* listed;
    int32_t* app_key;
    int32_t* app_id;
    int32_t* name_id;
    uint8_t* is_executor;
    uint8_t* spark_scheduler;
    uint8_t* rr;                        // [n_app_keys] RR flag
};

struct OhTableLookup {
    const uint8_t* rr;
    OhtSet S;
    const int32_t* row_of_node;
    __device__ int32_t row(int32_t node) const { return row_of_node[node]; }
    __device__ bool has(int32_t ak, int32_t ai, int32_t nm, bool exe, bool* rr_exists) const {
        uint32_t at;
        *rr_exists = rr[ak] != 0;
        if (*rr_exists && oht_find(S, oht_key(0, ak, nm), &at)) return true;
        return exe && oht_find(S, oht_key(1, ai, nm), &at);
    }
};

// One update, staged on the device; optional columns are NULL as in gp_overhead_delta
struct OhtDelta {
    long long n_write;
    int32_t n_rr;
    long long n_member;
    int32_t n_slots, n_node_ids, n_app_keys, n_app_ids, n_names;
    const int32_t* slot;
    const int32_t* node_id;
    const long long* req[3];
    const uint8_t* listed;
    const int32_t* app_key;
    const int32_t* app_id;
    const int32_t* name_id;
    const uint8_t* is_executor;
    const uint8_t* spark_scheduler;
    const int32_t* rr_app_key;
    const uint8_t* rr_exists;
    const uint8_t* member_kind;
    const int32_t* member_app;
    const int32_t* member_name;
    const uint8_t* member_present;
};

// Update bookkeeping, read back with the error word: cells claimed and tombstones written by this update
struct OhtWord { int err, unused; unsigned long long inserted, removed; };

// Duplicates: slots and app keys through per-table stamps (stamped_twice); member triples through a scratch set of the delta's
// keys.
static __global__ void gp_oht_check(OhtDelta D, uint32_t* slot_stamp, uint32_t* rr_stamp, uint32_t seq, OhtSet dup, OhtWord* w) {
    const long long total = D.n_write + D.n_rr + D.n_member;
    int bad = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        if (i < D.n_write) {
            const int32_t s = D.slot[i], node = D.node_id[i];
            if (s < 0 || s >= D.n_slots) { bad |= kOhtErrRange; continue; }
            if (stamped_twice(slot_stamp + s, seq)) bad |= kOhtErrDuplicate;
            if (node == -1) continue;                                  // a free slot: nothing else is read
            if (node < 0 || node >= D.n_node_ids) bad |= kOhtErrRange;
            for (int d = 0; d < 3; ++d) {
                const long long q = D.req[d] ? D.req[d][i] : 0;
                if (q < 0) bad |= kOhtErrNegative;
                else if (q >= kMaxQuantity) bad |= kOhtErrRequest;
            }
            if (D.listed && !D.listed[i]) continue;                    // the pod fields are not read
            const int32_t ak = D.app_key[i], ai = D.app_id[i], nm = D.name_id[i];
            if (ak < -1 || ak >= D.n_app_keys || ai < -1 || ai >= D.n_app_ids || nm < 0 || nm >= D.n_names) bad |= kOhtErrRange;
            else if ((ak < 0) != (ai < 0)) bad |= kOhtErrAppPair;
        } else if (i < D.n_write + D.n_rr) {
            const int32_t k = D.rr_app_key[i - D.n_write];
            if (k < 0 || k >= D.n_app_keys) { bad |= kOhtErrRange; continue; }
            if (stamped_twice(rr_stamp + k, seq)) bad |= kOhtErrDuplicate;
        } else {
            const long long m = i - D.n_write - D.n_rr;
            const int kind = D.member_kind[m];
            const int32_t app = D.member_app[m], nm = D.member_name[m];
            if (kind > 1 || app < 0 || app >= (kind ? D.n_app_ids : D.n_app_keys) || nm < 0 || nm >= D.n_names) { bad |= kOhtErrRange; continue; }
            const unsigned long long k = oht_key(kind, app, nm);
            for (uint32_t h = oh_hash(k) & dup.mask;; h = (h + 1) & dup.mask) {
                const unsigned long long prev = atomicCAS(dup.cell + h, kOhEmpty, k);
                if (prev == kOhEmpty) break;
                if (prev == k) { bad |= kOhtErrDuplicate; break; }
            }
        }
    }
    if (bad) atomicOr(&w->err, bad);
}

static __global__ void gp_oht_rehash(OhtSet from, OhtSet to) {
    for (long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x; h <= (long long)from.mask; h += (long long)gridDim.x * blockDim.x) {
        const unsigned long long k = from.cell[h];
        if (k != kOhEmpty && k != kOhTomb) oht_claim(to, k);
    }
}

static __global__ void gp_oht_apply(OhtDelta D, OhtCols T, OhtSet S, OhtWord* w) {
    if (*(volatile int*)&w->err) return;
    const long long total = D.n_write + D.n_rr + D.n_member;
    unsigned long long removed = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        if (i < D.n_write) {
            const int32_t s = D.slot[i];
            T.node_id[s] = D.node_id[i];
            for (int d = 0; d < 3; ++d) T.req[d][s] = D.req[d] ? D.req[d][i] : 0;
            T.listed[s] = D.listed ? D.listed[i] : 1;
            T.app_key[s] = D.app_key[i];
            T.app_id[s] = D.app_id[i];
            T.name_id[s] = D.name_id[i];
            T.is_executor[s] = D.is_executor ? D.is_executor[i] : 0;
            T.spark_scheduler[s] = D.spark_scheduler ? D.spark_scheduler[i] : 0;
        } else if (i < D.n_write + D.n_rr) {
            const long long r = i - D.n_write;
            T.rr[D.rr_app_key[r]] = D.rr_exists[r] ? 1 : 0;
        } else {
            const long long m = i - D.n_write - D.n_rr;
            uint32_t at;
            if (!D.member_present[m] && oht_find(S, oht_key(D.member_kind[m], D.member_app[m], D.member_name[m]), &at)) {
                S.cell[at] = kOhTomb;
                ++removed;
            }
        }
    }
    if (removed) atomicAdd(&w->removed, removed);
}

static __global__ void gp_oht_insert(OhtDelta D, OhtSet S, OhtWord* w) {
    if (*(volatile int*)&w->err) return;
    unsigned long long inserted = 0;
    for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < D.n_member; m += (long long)gridDim.x * blockDim.x) {
        if (!D.member_present[m]) continue;
        const unsigned long long k = oht_key(D.member_kind[m], D.member_app[m], D.member_name[m]);
        uint32_t at;
        if (oht_find(S, k, &at)) continue;                          // present already: a no-op
        oht_claim(S, k);
        ++inserted;
    }
    if (inserted) atomicAdd(&w->inserted, inserted);
}

}  // namespace gp

// gangpack_labels.cuh -- how device code reads the resident label table (gangpack_label_table.cu): a node's labels as a
// range of one key column and one value column, and the lookup of a key in that range.  Shared by the affinity match
// (gangpack_affinity.cuh) and the node-table entries' gather (gangpack_node_table.cu); device functions only.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace gp {

// The label table's rows: node i's labels are entries [r * stride, r * stride + count[r]) of key / val, r = node_id[i]; an id
// outside [0, n_rows) reads as no labels (gp_aff_ids refuses it)
struct AffLabelsResident {
    int32_t n, n_rows, stride;
    const int32_t* node_id;               // [n]
    const int32_t* count;                 // [n_rows]
    const int32_t* key;                   // [n_rows * stride]
    const int32_t* val;
    const uint8_t* val_int_ok;            // [n_values] ParseInt of the value succeeded
    const long long* val_int;             // [n_values]
    __device__ __forceinline__ void range(int32_t node, long long& lo, long long& hi) const {
        const int32_t r = node_id[node];
        lo = hi = 0;
        if (r >= 0 && r < n_rows) { lo = (long long)r * stride; hi = lo + count[r]; }
    }
    __device__ __forceinline__ bool int_at(long long e, long long& v) const {
        const int32_t x = val[e];
        if (!val_int_ok[x]) return false;
        v = val_int[x];
        return true;
    }
};

// position of key k in the sorted keys[lo, hi), or -1
__device__ __forceinline__ long long aff_find(const int32_t* __restrict__ keys, long long lo, long long hi, int32_t k) {
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        const int32_t v = keys[mid];
        if (v == k) return mid;
        if (v < k) lo = mid + 1; else hi = mid;
    }
    return -1;
}

}  // namespace gp

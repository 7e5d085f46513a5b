// gangpack_tilesort.cuh -- the sort primitive of gangpack_sort.cuh: tiles sorted in shared memory, ranks by binary search
// across tiles (see there).  Templates only, so that any translation unit may instantiate them for its own key: a key type
// K needs key_less(K, K), a strict total order, and key_max(const K*), a key above every real one.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace gp {

// ---- sort primitive: tiles sorted in shared memory, ranks by binary search across tiles ---------------------------
constexpr int kSortTile = 4096;
constexpr int kSortThreads = 1024;

// (1) sorted[tile] = the tile's keys in ascending order.  count_ptr: the number of keys lives on the device (candidate
// lists) or is `n` when NULL.  Dynamic shared memory: kSortTile * sizeof(K).
template <class K>
__global__ void __launch_bounds__(kSortThreads) gp_sort_tiles(int32_t n, const int32_t* __restrict__ count_ptr, const K* __restrict__ keys,
                                                              K* __restrict__ sorted) {
    extern __shared__ __align__(16) unsigned char sort_smem[];
    K* t = reinterpret_cast<K*>(sort_smem);
    if (count_ptr) n = *count_ptr;
    const int32_t base = blockIdx.x * kSortTile;
    if (base >= n) return;
    const int32_t m = min(kSortTile, n - base);
    for (int32_t i = threadIdx.x; i < kSortTile; i += blockDim.x) t[i] = i < m ? keys[base + i] : key_max((const K*)nullptr);
    __syncthreads();
    for (int32_t size = 2; size <= kSortTile; size <<= 1) {
        for (int32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (int32_t p = threadIdx.x; p < kSortTile / 2; p += blockDim.x) {
                const int32_t lo = 2 * p - (p & (stride - 1));          // index with bit `stride` clear
                const int32_t hi = lo + stride;
                const bool up = (lo & size) == 0;
                const K a = t[lo], b = t[hi];
                if (key_less(b, a) == up) { t[lo] = b; t[hi] = a; }
            }
            __syncthreads();
        }
    }
    for (int32_t i = threadIdx.x; i < m; i += blockDim.x) sorted[base + i] = t[i];
}

// (2) pos[i] = #{ j : key_j < key_i } = sum over tiles of lower_bound(tile, key_i)
template <class K>
__global__ void __launch_bounds__(256) gp_rank_by_search(int32_t n, const int32_t* __restrict__ count_ptr, const K* __restrict__ keys,
                                                         const K* __restrict__ sorted, int32_t* __restrict__ pos) {
    if (count_ptr) n = *count_ptr;
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const K me = keys[i];
    int32_t cnt = 0;
    for (int32_t base = 0; base < n; base += kSortTile) {
        const K* t = sorted + base;
        int32_t lo = 0, hi = min(kSortTile, n - base);              // first index whose key is not < me
        while (lo < hi) {
            const int32_t mid = (lo + hi) >> 1;
            if (key_less(t[mid], me)) lo = mid + 1; else hi = mid;
        }
        cnt += lo;
    }
    pos[i] = cnt;
}

}  // namespace gp

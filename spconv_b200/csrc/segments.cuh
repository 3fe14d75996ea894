// Keyed row grouping, the step in front of the segment kernels: rows get a small integer key, a stable argsort orders
// them, and segment k is the sorted positions [offsets[k], offsets[k+1]), in ascending row order.  Offsets take one
// binary search per segment, not one thread per key filling the gap up to the next key: with a host-known bound,
// segments [M, bound) are all empty, and one thread would write that whole gap serially.
#pragma once
#include "common.cuh"

namespace spx {

// ---------------------------------------------------------------- host
// stable radix argsort of one or two key arrays (sort.cu): keys sorted in place, argsort receives the order
size_t radix_argsort_workspace_bytes(int64_t n);
int radix_argsort_pair(uint32_t *mask0, int32_t *argsort0, int64_t n0, uint32_t *mask1, int32_t *argsort1, int64_t n1,
                       int key_bits, void *ws0, size_t ws0_bytes, void *ws1, size_t ws1_bytes, cudaStream_t stream);

// key width of a sort over the keys 0..max_key: the least b >= 1 with max_key < 2^b, at most 32
inline int sort_key_bits(int64_t max_key) {
    int b = 1;
    while (b < 32 && (max_key >> b) != 0) ++b;
    return b;
}

// temp bytes of cub::DeviceRadixSort::SortPairs over n uint32 pairs, never below a floor covering its buffers
size_t cub_sort_pairs_temp_bytes(int64_t n);
// stable argsort of keys [n] in 0..max_key: keys sorted in place, order [n]; sort_ws of radix_argsort_workspace_bytes(n)
int sort_by_key(uint32_t *keys, int64_t n, int64_t max_key, int32_t *order, void *sort_ws, size_t sort_ws_bytes,
                cudaStream_t stream);
// offsets [m + 1] of sorted_keys [n]: offsets[k] = first position whose key is >= k, for k = 0..m
int segment_offsets(const uint32_t *sorted_keys, int64_t n, int64_t m, int32_t *offsets, cudaStream_t stream);
// keys -> sort -> segments of the rows of dst [rows] (sparse_add.cu): order [rows], offsets [M + 1]
int group_rows(const int32_t *dst, int64_t rows, int64_t M, int32_t *order, int32_t *offsets, void *workspace,
               size_t workspace_bytes, cudaStream_t stream, const char *who);
// the fp32 sum of every segment of x [rows, channels] in sorted order (sparse_add.cu, one operand)
int sum_segments(const void *x, int64_t rows, const int32_t *order, const int32_t *offsets, int64_t M, int channels,
                 int dtype, void *out, cudaStream_t stream);
// keys -> sort -> per-sample segments cut into chunks of GP_CHUNK rows (global_pool.cu)
int group_samples(const int32_t *coords, int64_t rows, int row_ints, int batch_size, const int32_t *num_valid,
                  uint32_t *keys, int32_t *order, void *sort_ws, int32_t *offsets, int32_t *cstart, int32_t *count,
                  cudaStream_t stream);

#ifdef __CUDACC__
// ---------------------------------------------------------------- device: searches over sorted arrays
// Each call site keeps its own widths: I is the index type, the comparison is the one of K (S) against X.
// first position p in [0, n) with keys[p] >= x (keys ascending), n when there is none
template <typename I, typename K, typename X>
__device__ __forceinline__ I first_at_least(const K *keys, I n, X x) {
    I lo = 0, hi = n;
    while (lo < hi) {
        const I mid = (lo + hi) >> 1;
        if (keys[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// the last i in [0, count) with start[i] <= x (start non-decreasing), 0 when there is none.  start is read through
// __ldg, so it must be global memory: an operand table in the kernel parameters keeps its own loop (sparse_add.cu).
template <typename I, typename S, typename X>
__device__ __forceinline__ I last_at_most(const S *start, I count, X x) {
    I lo = 0, hi = count - 1;
    while (lo < hi) {
        const I mid = (lo + hi + 1) >> 1;
        if (__ldg(start + mid) <= x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}
#endif

}  // namespace spx

// Ranking a set of DISTINCT 32-bit payloads in [0, n) without a sort: the rank of payload p is the
// number of payloads below p = the number of set bits below p in a bitmap over [0, n).
//   mark:   one atomicOr per payload, plus a count per 1024-bit tile (rank_mark);
//   prefix: the LAST block of the marking kernel to finish turns the tile counts into an exclusive
//           prefix (rank_prefix_last_block), so no separate scan launch is needed;
//   rank:   tile prefix + popcount of at most 32 words (rank_of), in a later kernel.
// Used by the regular-conv rulebook (payload = the first (offset, input) pair that touched an output,
// rulebook.cu) and by the hash table (payload = the insertion ordinal of a key, hash_table.cu).
#pragma once
#include "common.cuh"

namespace spx {

constexpr int RANK_TILE_WORDS = 32;              // bitmap words per counted tile (1024 payloads)

// bitmap words, then the tile counts; the caller zeroes both (and its completion counter) before marking
static inline size_t rank_scratch_bytes(int64_t n, int64_t *ntiles = nullptr) {
    const int64_t words = div_up64(n > 0 ? n : 1, 32), tiles = div_up64(words, RANK_TILE_WORDS);
    if (ntiles) *ntiles = tiles;
    return align_up((size_t)(tiles * RANK_TILE_WORDS + tiles + 1) * 4, 256);
}

#ifdef __CUDACC__

__device__ __forceinline__ void rank_mark(uint32_t p, uint32_t *__restrict__ bitmap, int *__restrict__ tile_cnt) {
    atomicOr(&bitmap[p >> 5], 1u << (p & 31));
    atomicAdd(&tile_cnt[p >> 10], 1);
}

// Called by every thread of every block of the marking kernel after its rank_mark calls (blockDim.x ==
// THREADS).  The last block to arrive (counted in *done, zero before the launch) rewrites tile_cnt as an
// exclusive prefix and returns true with *total = the number of marked payloads; every other block
// returns false.
template <int THREADS>
__device__ __forceinline__ bool rank_prefix_last_block(int *__restrict__ tile_cnt, int64_t tiles, int *__restrict__ done,
                                                       int *total) {
    __shared__ int warp_sums[THREADS / 32];
    __shared__ int carry_s, last_s;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) { last_s = atomicAdd(done, 1) == (int)gridDim.x - 1; carry_s = 0; }
    __syncthreads();
    if (!last_s) return false;
    __threadfence();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t t0 = 0; t0 < tiles; t0 += THREADS) {
        const int64_t t = t0 + threadIdx.x;
        const int v = t < tiles ? __ldcg(tile_cnt + t) : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        int wbase = 0;
        for (int w = 0; w < warp; ++w) wbase += warp_sums[w];
        const int carry = carry_s;
        if (t < tiles) tile_cnt[t] = carry + wbase + incl - v;
        __syncthreads();
        if (threadIdx.x == THREADS - 1) carry_s = carry + wbase + incl;
        __syncthreads();
    }
    *total = carry_s;
    return true;
}

// rank of a marked payload p once the prefix is in place
__device__ __forceinline__ int rank_of(uint32_t p, const uint32_t *__restrict__ bitmap, const int *__restrict__ tile_prefix) {
    const uint32_t word = p >> 5, first = word & ~(uint32_t)(RANK_TILE_WORDS - 1);
    int r = __ldg(tile_prefix + (p >> 10)) + __popc(__ldg(bitmap + word) & ((1u << (p & 31)) - 1u));
    for (uint32_t wd = first; wd < word; ++wd) r += __popc(__ldg(bitmap + wd));
    return r;
}

#endif  // __CUDACC__

}  // namespace spx

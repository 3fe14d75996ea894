// Fixed-size GPU hash table behind spconv_b200.pytorch.hash.HashTable (reference API:
// spconv/pytorch/hash.py; semantics: the CPU tsl::robin_map branch of spconv/csrc/hash/core.py).
//
// Storage is split: keys [cap] and values [cap] are the user-visible keys_data / values_data; a key of
// 4 or 8 bytes is claimed with a CAS, a value of 4 or 8 bytes is moved as raw bits (NaN payloads and
// -0.0 survive).  The largest value of the signed key type marks an empty slot, so that key is never
// stored.  The slot of a key is the multiply-high reduction of mix32 / mix64 onto [0, cap) (cap need
// not be a power of two), then linear probing with wrap-around.  The caller keeps the number of keys
// inserted so far below cap, so there is always an empty slot and every probe chain ends.
//
// Every result is deterministic:
//   first [cap]  insertion ordinal of the key in the slot (call base + position), INT32_MAX = none.
//                insert: atomicMin, then only the thread whose ordinal survived writes its value, so
//                the FIRST insertion of a key wins (later duplicates and re-inserts change nothing);
//   tag [cap]    (epoch << 32 | position) of the last insert_exist_keys write: atomicMax, then only the
//                winning thread writes, so the LAST occurrence in a call wins.  Tags of older calls are
//                smaller, so the array is never reset;
//   rank         items / assign_arange_ number the keys in first-insertion order: the ordinals are
//                distinct, so they are ranked with the bitmap / tile-prefix / popcount scheme of
//                rank.cuh (no sort).  The count is written on the device.
#include "common.cuh"
#include "hash.cuh"
#include "rank.cuh"

namespace spx {

constexpr int HT_THREADS = 256;
constexpr int32_t HT_NONE = 2147483647;          // first[] of a slot that holds no key

template <typename K> struct HtKey;
template <> struct HtKey<unsigned int> {
    static constexpr unsigned int EMPTY = 0x7FFFFFFFu;                       // INT32_MAX
    __device__ __forceinline__ static uint32_t hash(unsigned int k) { return mix32(k); }
};
template <> struct HtKey<unsigned long long> {
    static constexpr unsigned long long EMPTY = 0x7FFFFFFFFFFFFFFFull;       // INT64_MAX
    __device__ __forceinline__ static uint32_t hash(unsigned long long k) { return mix64(k); }
};

template <typename K> __device__ __forceinline__ uint32_t home_slot(K key, uint32_t cap) {
    return (uint32_t)(((uint64_t)HtKey<K>::hash(key) * cap) >> 32);
}

// read-only probe: slot of key, or -1
template <typename K> __device__ __forceinline__ int32_t find_slot(const K *__restrict__ tkeys, uint32_t cap, K key) {
    if (key == HtKey<K>::EMPTY) return -1;
    uint32_t s = home_slot(key, cap);
    while (true) {
        const K cur = tkeys[s];
        if (cur == key) return (int32_t)s;
        if (cur == HtKey<K>::EMPTY) return -1;
        if (++s == cap) s = 0;
    }
}

template <typename K, typename V>
__global__ void ht_clear_kernel(K *__restrict__ tkeys, V *__restrict__ tvals, int32_t *__restrict__ first,
                                unsigned long long *__restrict__ tag, uint32_t cap) {
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += stride) {
        tkeys[s] = HtKey<K>::EMPTY;
        tvals[s] = 0;
        first[s] = HT_NONE;
        tag[s] = 0ull;
    }
}

// insert, launch 1: claim or find the slot, keep the smallest ordinal in first[], remember the slot
template <typename K>
__global__ void __launch_bounds__(HT_THREADS)
ht_insert_claim_kernel(K *__restrict__ tkeys, int32_t *__restrict__ first, uint32_t cap, const K *__restrict__ keys,
                       int32_t n, int32_t base, int32_t *__restrict__ slot_of) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const K key = __ldg(keys + i);
    int32_t slot = -1;
    if (key != HtKey<K>::EMPTY) {
        uint32_t s = home_slot(key, cap);
        while (true) {
            K cur = *(volatile K *)(tkeys + s);
            if (cur == HtKey<K>::EMPTY) cur = atomicCAS(tkeys + s, HtKey<K>::EMPTY, key);
            if (cur == HtKey<K>::EMPTY || cur == key) break;
            if (++s == cap) s = 0;
        }
        atomicMin(first + s, (int32_t)(base + i));
        slot = (int32_t)s;
    }
    slot_of[i] = slot;
}

// insert, launch 2: the thread whose ordinal is the slot's first writes its value (0 without values)
template <typename V>
__global__ void __launch_bounds__(HT_THREADS)
ht_insert_value_kernel(V *__restrict__ tvals, const int32_t *__restrict__ first, const V *__restrict__ values,
                       int32_t n, int32_t base, const int32_t *__restrict__ slot_of) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t s = slot_of[i];
    if (s < 0 || first[s] != base + i) return;
    tvals[s] = values ? __ldg(values + i) : (V)0;
}

template <typename K, typename V>
__global__ void __launch_bounds__(HT_THREADS)
ht_query_kernel(const K *__restrict__ tkeys, const V *__restrict__ tvals, uint32_t cap, const K *__restrict__ keys,
                int32_t n, V *__restrict__ values, uint8_t *__restrict__ is_empty) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t s = find_slot(tkeys, cap, __ldg(keys + i));
    if (s >= 0) values[i] = tvals[s];
    is_empty[i] = s < 0;
}

// insert_exist_keys, launch 1: find the slot, keep the largest (epoch, position) tag
template <typename K>
__global__ void __launch_bounds__(HT_THREADS)
ht_exist_claim_kernel(const K *__restrict__ tkeys, unsigned long long *__restrict__ tag, uint32_t cap,
                      const K *__restrict__ keys, int32_t n, unsigned long long epoch, int32_t *__restrict__ slot_of,
                      uint8_t *__restrict__ is_empty) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t s = find_slot(tkeys, cap, __ldg(keys + i));
    if (s >= 0) atomicMax(tag + s, (epoch << 32) | (uint32_t)i);
    slot_of[i] = s;
    is_empty[i] = s < 0;
}

// insert_exist_keys, launch 2: the last occurrence of every found key writes its value
template <typename V>
__global__ void __launch_bounds__(HT_THREADS)
ht_exist_value_kernel(V *__restrict__ tvals, const unsigned long long *__restrict__ tag, const V *__restrict__ values,
                      int32_t n, unsigned long long epoch, const int32_t *__restrict__ slot_of) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t s = slot_of[i];
    if (s < 0 || tag[s] != ((epoch << 32) | (uint32_t)i)) return;
    tvals[s] = __ldg(values + i);
}

// rank, launch 1: mark the ordinal of every stored key; the last block builds the tile prefix and
// writes the count (C = the unsigned type of the key's size, as in the reference)
template <typename C>
__global__ void __launch_bounds__(HT_THREADS)
ht_mark_kernel(const int32_t *__restrict__ first, uint32_t cap, uint32_t *__restrict__ bitmap, int *__restrict__ tile_cnt,
               int64_t tiles, int *__restrict__ done, C *__restrict__ count) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < cap) {
        const int32_t f = first[s];
        if (f != HT_NONE) rank_mark((uint32_t)f, bitmap, tile_cnt);
    }
    int total;
    if (rank_prefix_last_block<HT_THREADS>(tile_cnt, tiles, done, &total) && threadIdx.x == 0) *count = (C)total;
}

// rank, launch 2: r = rank of the slot's ordinal; assign_arange_: value = r; items: row r = (key, value)
template <typename K, typename V>
__global__ void __launch_bounds__(HT_THREADS)
ht_rank_kernel(const K *__restrict__ tkeys, V *__restrict__ tvals, const int32_t *__restrict__ first, uint32_t cap,
               const uint32_t *__restrict__ bitmap, const int *__restrict__ tile_prefix, int assign,
               K *__restrict__ out_keys, V *__restrict__ out_values, int64_t out_rows) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= cap) return;
    const int32_t f = first[s];
    if (f == HT_NONE) return;
    const int r = rank_of((uint32_t)f, bitmap, tile_prefix);
    if (assign) {
        tvals[s] = (V)r;
    } else if (r < out_rows) {
        out_keys[r] = tkeys[s];
        out_values[r] = tvals[s];
    }
}

static unsigned ht_blocks(int64_t n) { return (unsigned)div_up64(n > 0 ? n : 1, HT_THREADS); }

static int check_table(int64_t max_size, int key_size, int value_size, const char *who) {
    SPX_REQUIRE(key_size == 4 || key_size == 8, "%s: key itemsize must be 4 or 8, got %d", who, key_size);
    SPX_REQUIRE(value_size == 4 || value_size == 8, "%s: value itemsize must be 4 or 8, got %d", who, value_size);
    SPX_REQUIRE(max_size >= 1 && max_size <= 2147483647ll, "%s: max_size %lld not in [1, 2^31 - 1]", who,
                (long long)max_size);
    return 0;
}

static int check_count(int64_t n, const char *who) {
    SPX_REQUIRE(n >= 0 && n <= 2147483647ll, "%s: key count %lld not in [0, 2^31 - 1]", who, (long long)n);
    return 0;
}

template <typename K, typename V>
static int launch_clear(void *tkeys, void *tvals, int32_t *first, uint64_t *tag, uint32_t cap, cudaStream_t stream) {
    const int64_t need = div_up64(cap, HT_THREADS), most = (int64_t)sm_count() * 8;
    const unsigned blocks = (unsigned)(need < most ? need : most);
    ht_clear_kernel<K, V><<<blocks, HT_THREADS, 0, stream>>>((K *)tkeys, (V *)tvals, first, (unsigned long long *)tag, cap);
    SPX_CHECK_LAUNCH("ht_clear_kernel");
    return 0;
}

template <typename K, typename V>
static int launch_query(const void *tkeys, const void *tvals, uint32_t cap, const void *keys, int32_t n, void *values,
                        uint8_t *is_empty, cudaStream_t stream) {
    ht_query_kernel<K, V><<<ht_blocks(n), HT_THREADS, 0, stream>>>((const K *)tkeys, (const V *)tvals, cap,
                                                                   (const K *)keys, n, (V *)values, is_empty);
    SPX_CHECK_LAUNCH("ht_query_kernel");
    return 0;
}

template <typename K, typename V>
static int launch_rank(const void *tkeys, void *tvals, const int32_t *first, uint32_t cap, uint32_t *bitmap,
                       int *tiles_cnt, int64_t ntiles, int *done, int assign, void *out_keys, void *out_values,
                       int64_t out_rows, void *count, cudaStream_t stream) {
    ht_mark_kernel<K><<<ht_blocks(cap), HT_THREADS, 0, stream>>>(first, cap, bitmap, tiles_cnt, ntiles, done, (K *)count);
    SPX_CHECK_LAUNCH("ht_mark_kernel");
    ht_rank_kernel<K, V><<<ht_blocks(cap), HT_THREADS, 0, stream>>>((const K *)tkeys, (V *)tvals, first, cap, bitmap,
                                                                    tiles_cnt, assign, (K *)out_keys, (V *)out_values,
                                                                    out_rows);
    SPX_CHECK_LAUNCH("ht_rank_kernel");
    return 0;
}

typedef unsigned int U4;
typedef unsigned long long U8;

// calls F<K, V>(args...) for the (key_size, value_size) pair
#define HT_DISPATCH(F, key_size, value_size, ...)                                                       \
    ((key_size) == 4 ? ((value_size) == 4 ? F<U4, U4>(__VA_ARGS__) : F<U4, U8>(__VA_ARGS__))           \
                     : ((value_size) == 4 ? F<U8, U4>(__VA_ARGS__) : F<U8, U8>(__VA_ARGS__)))

}  // namespace spx

using namespace spx;

extern "C" size_t spx_hash_workspace_size(int64_t num_keys, int64_t ordinal_count) {
    if (num_keys < 0 || ordinal_count < 0) return 0;
    return align_up((size_t)num_keys * 4, 256) + rank_scratch_bytes(ordinal_count) + 2 * 256;
}

extern "C" int spx_hash_clear(void *table_keys, void *table_values, int32_t *first, uint64_t *tag, int64_t max_size,
                              int key_size, int value_size, spx_stream_t stream_) {
    if (int rc = check_table(max_size, key_size, value_size, "hash_clear")) return rc;
    SPX_REQUIRE(table_keys && table_values && first && tag, "hash_clear: NULL pointer argument");
    return HT_DISPATCH(launch_clear, key_size, value_size, table_keys, table_values, first, tag, (uint32_t)max_size,
                       (cudaStream_t)stream_);
}

template <typename K, typename V>
static int launch_insert(void *tkeys, void *tvals, int32_t *first, uint32_t cap, const void *keys, const void *values,
                         int32_t n, int32_t base, int32_t *slot_of, cudaStream_t stream) {
    ht_insert_claim_kernel<K><<<ht_blocks(n), HT_THREADS, 0, stream>>>((K *)tkeys, first, cap, (const K *)keys, n, base,
                                                                       slot_of);
    SPX_CHECK_LAUNCH("ht_insert_claim_kernel");
    ht_insert_value_kernel<V><<<ht_blocks(n), HT_THREADS, 0, stream>>>((V *)tvals, first, (const V *)values, n, base,
                                                                       slot_of);
    SPX_CHECK_LAUNCH("ht_insert_value_kernel");
    return 0;
}

extern "C" int spx_hash_insert(void *table_keys, void *table_values, int32_t *first, int64_t max_size, int key_size,
                               int value_size, const void *keys, const void *values, int64_t n, int64_t ordinal_base,
                               void *workspace, size_t workspace_bytes, spx_stream_t stream_) {
    if (int rc = check_table(max_size, key_size, value_size, "hash_insert")) return rc;
    if (int rc = check_count(n, "hash_insert")) return rc;
    SPX_REQUIRE(ordinal_base >= 0 && ordinal_base + n < max_size,
                "hash_insert: inserted count exceed maximum hash size (%lld + %lld keys, max_size %lld)",
                (long long)ordinal_base, (long long)n, (long long)max_size);
    if (n == 0) return 0;
    SPX_REQUIRE(table_keys && table_values && first && keys && workspace, "hash_insert: NULL pointer argument");
    SPX_REQUIRE(workspace_bytes >= spx_hash_workspace_size(n, 0), "hash_insert: workspace too small: need %zu, have %zu",
                spx_hash_workspace_size(n, 0), workspace_bytes);
    return HT_DISPATCH(launch_insert, key_size, value_size, table_keys, table_values, first, (uint32_t)max_size, keys,
                       values, (int32_t)n, (int32_t)ordinal_base, (int32_t *)workspace, (cudaStream_t)stream_);
}

extern "C" int spx_hash_query(const void *table_keys, const void *table_values, int64_t max_size, int key_size,
                              int value_size, const void *keys, void *values, uint8_t *is_empty, int64_t n,
                              spx_stream_t stream_) {
    if (int rc = check_table(max_size, key_size, value_size, "hash_query")) return rc;
    if (int rc = check_count(n, "hash_query")) return rc;
    if (n == 0) return 0;
    SPX_REQUIRE(table_keys && table_values && keys && values && is_empty, "hash_query: NULL pointer argument");
    return HT_DISPATCH(launch_query, key_size, value_size, table_keys, table_values, (uint32_t)max_size, keys,
                       (int32_t)n, values, is_empty, (cudaStream_t)stream_);
}

template <typename K, typename V>
static int launch_exist(const void *tkeys, void *tvals, uint64_t *tag, uint32_t cap, const void *keys, const void *values,
                        int32_t n, unsigned long long epoch, uint8_t *is_empty, int32_t *slot_of, cudaStream_t stream) {
    ht_exist_claim_kernel<K><<<ht_blocks(n), HT_THREADS, 0, stream>>>((const K *)tkeys, (unsigned long long *)tag, cap,
                                                                      (const K *)keys, n, epoch, slot_of, is_empty);
    SPX_CHECK_LAUNCH("ht_exist_claim_kernel");
    ht_exist_value_kernel<V><<<ht_blocks(n), HT_THREADS, 0, stream>>>((V *)tvals, (const unsigned long long *)tag,
                                                                      (const V *)values, n, epoch, slot_of);
    SPX_CHECK_LAUNCH("ht_exist_value_kernel");
    return 0;
}

extern "C" int spx_hash_insert_exist(const void *table_keys, void *table_values, uint64_t *tag, int64_t max_size,
                                     int key_size, int value_size, const void *keys, const void *values,
                                     uint8_t *is_empty, int64_t n, int64_t epoch, void *workspace,
                                     size_t workspace_bytes, spx_stream_t stream_) {
    if (int rc = check_table(max_size, key_size, value_size, "hash_insert_exist")) return rc;
    if (int rc = check_count(n, "hash_insert_exist")) return rc;
    SPX_REQUIRE(epoch >= 1 && epoch <= 4294967295ll, "hash_insert_exist: epoch %lld not in [1, 2^32 - 1]",
                (long long)epoch);
    if (n == 0) return 0;
    SPX_REQUIRE(table_keys && table_values && tag && keys && values && is_empty && workspace,
                "hash_insert_exist: NULL pointer argument");
    SPX_REQUIRE(workspace_bytes >= spx_hash_workspace_size(n, 0),
                "hash_insert_exist: workspace too small: need %zu, have %zu", spx_hash_workspace_size(n, 0),
                workspace_bytes);
    return HT_DISPATCH(launch_exist, key_size, value_size, table_keys, table_values, tag, (uint32_t)max_size, keys,
                       values, (int32_t)n, (unsigned long long)epoch, is_empty, (int32_t *)workspace,
                       (cudaStream_t)stream_);
}

extern "C" int spx_hash_rank(const void *table_keys, void *table_values, const int32_t *first, int64_t max_size,
                             int key_size, int value_size, int64_t ordinal_count, int assign, void *out_keys,
                             void *out_values, int64_t out_rows, void *count, void *workspace, size_t workspace_bytes,
                             spx_stream_t stream_) {
    if (int rc = check_table(max_size, key_size, value_size, "hash_rank")) return rc;
    SPX_REQUIRE(ordinal_count >= 0 && ordinal_count < max_size, "hash_rank: ordinal count %lld not in [0, %lld)",
                (long long)ordinal_count, (long long)max_size);
    SPX_REQUIRE(out_rows >= 0, "hash_rank: negative output row count");
    SPX_REQUIRE(count != nullptr, "hash_rank: count is NULL");
    SPX_REQUIRE(table_keys && table_values && first, "hash_rank: NULL pointer argument");
    SPX_REQUIRE(assign || out_rows == 0 || (out_keys && out_values), "hash_rank: NULL output pointer");
    cudaStream_t stream = (cudaStream_t)stream_;
    if (ordinal_count == 0) {                        // nothing was ever inserted
        SPX_CHECK_CUDA(cudaMemsetAsync(count, 0, key_size, stream));
        return 0;
    }
    SPX_REQUIRE(workspace != nullptr, "hash_rank: workspace is NULL");
    SPX_REQUIRE(workspace_bytes >= spx_hash_workspace_size(0, ordinal_count),
                "hash_rank: workspace too small: need %zu, have %zu", spx_hash_workspace_size(0, ordinal_count),
                workspace_bytes);
    int64_t ntiles = 0;
    const size_t rank_bytes = rank_scratch_bytes(ordinal_count, &ntiles);
    WorkspaceCarver ws(workspace, workspace_bytes);
    uint32_t *bitmap = (uint32_t *)ws.take<char>(rank_bytes);
    int *tile_cnt = (int *)(bitmap + ntiles * RANK_TILE_WORDS);
    int *done = ws.take<int>(1);
    SPX_CHECK_CUDA(cudaMemsetAsync(workspace, 0, ws.off, stream));    // bitmap, tile counts, completion counter
    return HT_DISPATCH(launch_rank, key_size, value_size, table_keys, table_values, first, (uint32_t)max_size, bitmap,
                       tile_cnt, ntiles, done, assign, out_keys, out_values, out_rows, count, stream);
}

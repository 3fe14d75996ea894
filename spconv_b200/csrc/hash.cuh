// Open-addressing hash tables shared by the rulebook kernels (rulebook.cu) and the point -> voxel
// front end (pointops.cu).  One packed 64-bit slot {key:32 | value:32} per entry for 32-bit keys so a
// probe is ONE 8-byte load (the reference probes split key / value arrays: "performance bound",
// spconv/csrc/sparse/indices.py:791); split arrays for 64-bit keys.  insert_min keeps the SMALLEST
// value per key = "first touch wins", which is what makes every ordering decision deterministic.
#pragma once
#include "common.cuh"

namespace spx {

// ------------------------------------------------------------------ keys
// key of the coordinate c = (batch, c_1 .. c_ndim) in a grid of `dims`: row-major, batch outermost.  The SubM
// rulebook (rulebook.cu) and the voxel -> point interpolation (point_interp.cu) insert and find with it.
__device__ __forceinline__ int64_t linear_key(const int (&c)[SPX_MAX_NDIM + 1], const int *dims, int ndim) {
    int64_t k = c[0];
#pragma unroll
    for (int a = 0; a < SPX_MAX_NDIM; ++a) if (a < ndim) k = k * dims[a] + c[a + 1];
    return k;
}

// ------------------------------------------------------------------ hash tables
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x85ebca6bu; x ^= x >> 13; x *= 0xc2b2ae35u; x ^= x >> 16;
    return x;
}
__device__ __forceinline__ uint32_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return (uint32_t)x;
}

// 32-bit keys: one packed slot, key in the high word so that atomicMin on the slot is a
// min over the value for equal keys.
struct Table32 {
    unsigned long long *slots;
    uint32_t cap_mask;
    static constexpr unsigned long long EMPTY = ~0ull;
    __device__ __forceinline__ void insert_min(int64_t key64, int32_t val) const {
        uint32_t key = (uint32_t)key64;
        unsigned long long packed = ((unsigned long long)key << 32) | (uint32_t)val;
        uint32_t h = mix32(key) & cap_mask;
        while (true) {
            unsigned long long prev = atomicCAS(&slots[h], EMPTY, packed);
            if (prev == EMPTY) return;
            if ((uint32_t)(prev >> 32) == key) {
                if ((uint32_t)prev > (uint32_t)val) atomicMin(&slots[h], packed);
                return;
            }
            h = (h + 1) & cap_mask;
        }
    }
    // insert_min that also reports the slot and whether THIS call created the entry; gives up after
    // max_probes steps (returns -1): the caller sized the table optimistically and must re-run
    __device__ __forceinline__ int64_t insert_min_slot(int64_t key64, int32_t val, bool &created, int max_probes) const {
        uint32_t key = (uint32_t)key64;
        unsigned long long packed = ((unsigned long long)key << 32) | (uint32_t)val;
        uint32_t h = mix32(key) & cap_mask;
        created = false;
        for (int step = 0; step < max_probes; ++step) {
            unsigned long long prev = atomicCAS(&slots[h], EMPTY, packed);
            if (prev == EMPTY) { created = true; return h; }
            if ((uint32_t)(prev >> 32) == key) {
                if ((uint32_t)prev > (uint32_t)val) atomicMin(&slots[h], packed);
                return h;
            }
            h = (h + 1) & cap_mask;
        }
        return -1;
    }
    __device__ __forceinline__ int32_t value_at(uint32_t s) const { return (int32_t)(uint32_t)slots[s]; }
    __device__ __forceinline__ void clear_slot(uint32_t s) const { slots[s] = EMPTY; }
    // returns slot index or -1
    __device__ __forceinline__ int64_t find_slot(int64_t key64, int32_t &val) const {
        uint32_t key = (uint32_t)key64;
        uint32_t h = mix32(key) & cap_mask;
        while (true) {
            unsigned long long cur = __ldg(&slots[h]);
            if (cur == EMPTY) return -1;
            if ((uint32_t)(cur >> 32) == key) { val = (int32_t)(uint32_t)cur; return h; }
            h = (h + 1) & cap_mask;
        }
    }
    // find_slot one probe at a time (find_many): the first slot, then one step from slot h; true once the
    // search ends (val = the value, or -1 when the key is absent), else h moves to the next slot
    __device__ __forceinline__ uint32_t home(int64_t key64) const { return mix32((uint32_t)key64) & cap_mask; }
    __device__ __forceinline__ bool find_step(int64_t key64, uint32_t &h, int32_t &val) const {
        const unsigned long long cur = __ldg(&slots[h]);
        if (cur == EMPTY) { val = -1; return true; }
        if ((uint32_t)(cur >> 32) == (uint32_t)key64) { val = (int32_t)(uint32_t)cur; return true; }
        h = (h + 1) & cap_mask;
        return false;
    }
    __device__ __forceinline__ bool occupied(uint32_t s, int64_t &key, int32_t &val) const {
        unsigned long long cur = slots[s];
        if (cur == EMPTY) return false;
        key = (int64_t)(uint32_t)(cur >> 32);
        val = (int32_t)(uint32_t)cur;
        return true;
    }
    __device__ __forceinline__ void set_value(uint32_t s, int32_t val) const {
        unsigned long long cur = slots[s];
        slots[s] = (cur & 0xFFFFFFFF00000000ull) | (uint32_t)val;
    }
};

// 64-bit keys: split arrays (volume >= 2^31)
struct Table64 {
    long long *keys;   // EMPTY = -1
    int32_t *vals;     // initialised to INT_MAX
    uint32_t cap_mask;
    __device__ __forceinline__ void insert_min(int64_t key, int32_t val) const {
        uint32_t h = mix64((uint64_t)key) & cap_mask;
        while (true) {
            long long prev = (long long)atomicCAS((unsigned long long *)&keys[h], (unsigned long long)-1ll,
                                                  (unsigned long long)key);
            if (prev == -1ll || prev == key) { atomicMin(&vals[h], val); return; }
            h = (h + 1) & cap_mask;
        }
    }
    __device__ __forceinline__ int64_t insert_min_slot(int64_t key, int32_t val, bool &created, int max_probes) const {
        uint32_t h = mix64((uint64_t)key) & cap_mask;
        created = false;
        for (int step = 0; step < max_probes; ++step) {
            long long prev = (long long)atomicCAS((unsigned long long *)&keys[h], (unsigned long long)-1ll,
                                                  (unsigned long long)key);
            if (prev == -1ll || prev == key) { created = prev == -1ll; atomicMin(&vals[h], val); return h; }
            h = (h + 1) & cap_mask;
        }
        return -1;
    }
    __device__ __forceinline__ int32_t value_at(uint32_t s) const { return vals[s]; }
    __device__ __forceinline__ int64_t find_slot(int64_t key, int32_t &val) const {
        uint32_t h = mix64((uint64_t)key) & cap_mask;
        while (true) {
            long long cur = keys[h];
            if (cur == -1ll) return -1;
            if (cur == key) { val = vals[h]; return h; }
            h = (h + 1) & cap_mask;
        }
    }
    __device__ __forceinline__ uint32_t home(int64_t key) const { return mix64((uint64_t)key) & cap_mask; }
    __device__ __forceinline__ bool find_step(int64_t key, uint32_t &h, int32_t &val) const {
        const long long cur = keys[h];
        if (cur == -1ll) { val = -1; return true; }
        if (cur == key) { val = vals[h]; return true; }
        h = (h + 1) & cap_mask;
        return false;
    }
    __device__ __forceinline__ bool occupied(uint32_t s, int64_t &key, int32_t &val) const {
        long long cur = keys[s];
        if (cur == -1ll) return false;
        key = cur; val = vals[s];
        return true;
    }
    __device__ __forceinline__ void set_value(uint32_t s, int32_t val) const { vals[s] = val; }
    __device__ __forceinline__ void clear_slot(uint32_t s) const { keys[s] = -1ll; }
};

// K independent finds kept in flight together: each round, every unfinished key loads its next slot, so the loads
// of a round do not wait on each other (K find_slot calls in a row would walk the chains one after another).
// val[j] = the value of key[j], -1 when it is absent or live[j] is false.
template <int K, typename Table>
__device__ __forceinline__ void find_many(const Table &t, const int64_t (&key)[K], const bool (&live)[K],
                                          int32_t (&val)[K]) {
    uint32_t h[K];
    bool busy[K];
    bool any = false;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        val[j] = -1;
        busy[j] = live[j];
        h[j] = live[j] ? t.home(key[j]) : 0u;
        any = any || busy[j];
    }
    while (any) {
        any = false;
#pragma unroll
        for (int j = 0; j < K; ++j) {
            if (busy[j]) busy[j] = !t.find_step(key[j], h[j], val[j]);
            any = any || busy[j];
        }
    }
}

// Host side: call f with the table over `slots` (and, for 64-bit keys, `vals`), so that one launch sequence
// serves both key widths.  f returns 0 or an error code, which is passed on.
template <typename F>
int visit_table(bool i64, void *slots, int32_t *vals, uint32_t capacity, F &&f) {
    if (!i64) return f(Table32{(unsigned long long *)slots, capacity - 1});
    return f(Table64{(long long *)slots, vals, capacity - 1});
}

// load factor <= 0.25: with linear probing the expected miss chain is ~1.4 slots and -- what
// matters on a GPU -- the MAX chain over the 32 lanes of a warp stays ~2-3 (at 0.5 it was ~6
// dependent L2 round trips per probe, measured with ncu on the 100 k-voxel cloud)
static uint32_t table_capacity(int64_t n_items, int factor = 4) {
    uint64_t cap = 1024;
    while (cap < (uint64_t)n_items * factor) cap <<= 1;
    return (uint32_t)cap;
}

}  // namespace spx

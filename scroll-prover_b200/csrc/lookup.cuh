// The open-addressing set of a lookup table's usable rows (lookup.cu), shared with the miss probe of mock.cu.
//
// A slot holds a u32 row index; its key is always read back from table[row].  lookup_build_launch fills the set so that a
// value's slot ends up holding the FIRST usable row with that value, whatever order the threads run in.
#pragma once
#include "common.cuh"

namespace b200zk {

constexpr uint32_t LK_EMPTY = 0xFFFFFFFFu;

struct LkKey {
    uint4 a, b;
};
__device__ __forceinline__ LkKey lk_load(const Fr* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    return LkKey{q[0], q[1]};
}
__device__ __forceinline__ bool lk_eq(const LkKey& x, const LkKey& y) {
    return ((x.a.x ^ y.a.x) | (x.a.y ^ y.a.y) | (x.a.z ^ y.a.z) | (x.a.w ^ y.a.w) | (x.b.x ^ y.b.x) | (x.b.y ^ y.b.y) |
            (x.b.z ^ y.b.z) | (x.b.w ^ y.b.w)) == 0;
}
// all four 64-bit limbs mixed into the top `log_slots` bits (multiply-xorshift): the range tables of the chunk circuits are
// consecutive small integers, whose Montgomery limbs differ in every word, but the hash must not rely on that
__device__ __forceinline__ uint64_t lk_hash(const LkKey& k, uint32_t log_slots) {
    uint64_t l0 = ((uint64_t)k.a.y << 32) | k.a.x, l1 = ((uint64_t)k.a.w << 32) | k.a.z;
    uint64_t l2 = ((uint64_t)k.b.y << 32) | k.b.x, l3 = ((uint64_t)k.b.w << 32) | k.b.z;
    uint64_t h = l0 * 0x9E3779B97F4A7C15ull;
    h = (h ^ (h >> 29) ^ l1) * 0xBF58476D1CE4E5B9ull;
    h = (h ^ (h >> 31) ^ l2) * 0x94D049BB133111EBull;
    h = (h ^ (h >> 30) ^ l3) * 0x9E3779B97F4A7C15ull;
    h ^= h >> 32;
    return (h * 0xD6E8FEB86659FD93ull) >> (64 - log_slots);
}

// the table row holding `key`, or LK_EMPTY when no usable row does
__device__ __forceinline__ uint32_t lk_find(const LkKey& key, const Fr* table, const uint32_t* slots, uint32_t log_slots) {
    const uint64_t mask = (1ull << log_slots) - 1;
    for (uint64_t h = lk_hash(key, log_slots);; h = (h + 1) & mask) {
        const uint32_t cur = slots[h];
        if (cur == LK_EMPTY || lk_eq(lk_load(table + cur), key)) return cur;
    }
}

// slots for `usable` rows: a power of two >= 2 usable (load factor <= 1/2), at least 64
inline uint32_t lk_log_slots(uint64_t usable) {
    uint32_t log_slots = 6;
    while ((1ull << log_slots) < 2 * usable) ++log_slots;
    return log_slots;
}

inline uint32_t lk_blocks(b200zk_ctx* ctx, uint64_t n) {
    uint64_t want = (n + 255) / 256, cap = (uint64_t)ctx->sm_count * 16;
    if (want > cap) want = cap;
    return (uint32_t)(want ? want : 1);
}

// lookup.cu: inserts the usable rows of `table` into `slots` (2^log_slots entries, all LK_EMPTY beforehand) on the context stream
int32_t lookup_build_launch(b200zk_ctx* ctx, const Fr* table, uint64_t usable, uint32_t* slots, uint32_t log_slots);

}  // namespace b200zk

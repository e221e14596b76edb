// dev::MockProver::verify_par's three checks on the device (halo2_proofs 1.1.0 @ scroll-tech/halo2 e5ddf67, src/dev.rs): every
// check lists the cells that fail it, in ascending flat index.
//
//   mock_nonzero_kernel      a gate's values (or any Fr column): bit f = value f != 0
//   mock_lookup_miss_kernel  bit j * 2^k + i = input j's value at row i < usable is in no usable table row (the set of
//                            lookup.cu, built by lookup_build_launch)
//   mock_copy_kernel         bit c * 2^k + r = cell (c, r) differs from its successor cell next[c * 2^k + r] of the copy cycle;
//                            a successor outside the columns raises `bad` and is not read
//   mock_count_kernel        popcount of each tile of MOCK_TILE_WORDS mask words
//   mock_scan_kernel         one block: exclusive prefix sum of the tile counts, the total last
//   mock_scatter_kernel      every tile writes its set bits' indices from its offset on, stopping at cap
//
// The checks write a bit mask, one 32-bit word per warp step (__ballot_sync), so the mask is complete without atomics or a
// clear.  The compaction is tile counts -> scan -> scatter: the index list is fixed by the mask alone, whatever the schedule.
#include "lookup.cuh"

namespace b200zk {

constexpr uint32_t MOCK_THREADS = 256, MOCK_WORDS_PER_THREAD = 8, MOCK_TILE_WORDS = MOCK_THREADS * MOCK_WORDS_PER_THREAD;

__device__ __forceinline__ bool fr_nonzero(const Fr* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    const uint4 a = q[0], b = q[1];
    return (a.x | a.y | a.z | a.w | b.x | b.y | b.z | b.w) != 0;
}

// whole warps walk the flat indices [0, n) together, so that the ballot of a warp step is one mask word
#define MOCK_WARP_LOOP(n)                                                                                                   \
    const uint32_t lane = threadIdx.x & 31;                                                                                 \
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;                                                               \
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < (n); base += stride)

__global__ void __launch_bounds__(MOCK_THREADS) mock_nonzero_kernel(const Fr* values, uint64_t n, uint32_t* mask) {
    MOCK_WARP_LOOP(n) {
        const uint64_t f = base + lane;
        const uint32_t bits = __ballot_sync(0xFFFFFFFFu, f < n && fr_nonzero(values + f));
        if (lane == 0) mask[base >> 5] = bits;
    }
}

__global__ void __launch_bounds__(MOCK_THREADS) mock_lookup_miss_kernel(const Fr* const* inputs, uint32_t k, uint64_t total,
                                                                        const Fr* table, uint64_t usable, const uint32_t* slots,
                                                                        uint32_t log_slots, uint32_t* mask) {
    MOCK_WARP_LOOP(total) {
        const uint64_t f = base + lane, i = f & ((1ull << k) - 1);
        bool miss = false;
        if (f < total && i < usable) miss = lk_find(lk_load(inputs[f >> k] + i), table, slots, log_slots) == LK_EMPTY;
        const uint32_t bits = __ballot_sync(0xFFFFFFFFu, miss);
        if (lane == 0) mask[base >> 5] = bits;
    }
}

__global__ void __launch_bounds__(MOCK_THREADS) mock_copy_kernel(const Fr* const* cols, uint32_t k, uint64_t total, const uint64_t* next,
                                                                 uint32_t* mask, uint32_t* bad) {
    MOCK_WARP_LOOP(total) {
        const uint64_t f = base + lane, rmask = (1ull << k) - 1;
        bool differs = false;
        if (f < total) {
            const uint64_t g = next[f];
            if (g >= total) {
                *bad = 1;
            } else {
                differs = !lk_eq(lk_load(cols[f >> k] + (f & rmask)), lk_load(cols[g >> k] + (g & rmask)));
            }
        }
        const uint32_t bits = __ballot_sync(0xFFFFFFFFu, differs);
        if (lane == 0) mask[base >> 5] = bits;
    }
}

// inclusive sum over the block (blockDim.x a multiple of 32, at most 1024); `warp_sums` holds 32 entries
__device__ __forceinline__ unsigned long long block_inclusive_sum(unsigned long long v, unsigned long long* warp_sums) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (lane >= d) v += u;
    }
    if (lane == 31) warp_sums[warp] = v;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = lane < (blockDim.x >> 5) ? warp_sums[lane] : 0;
        for (uint32_t d = 1; d < 32; d <<= 1) {
            const unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, w, d);
            if (lane >= d) w += u;
        }
        warp_sums[lane] = w;
    }
    __syncthreads();
    const unsigned long long r = v + (warp ? warp_sums[warp - 1] : 0);
    __syncthreads();  // warp_sums may be reused by the caller's next round
    return r;
}

__global__ void __launch_bounds__(MOCK_THREADS) mock_count_kernel(const uint32_t* mask, uint64_t words, uint32_t* tile_counts) {
    __shared__ unsigned long long warp_sums[32];
    const uint64_t w0 = (uint64_t)blockIdx.x * MOCK_TILE_WORDS + (uint64_t)threadIdx.x * MOCK_WORDS_PER_THREAD;
    uint32_t c = 0;
    for (uint32_t w = 0; w < MOCK_WORDS_PER_THREAD; ++w)
        if (w0 + w < words) c += __popc(mask[w0 + w]);
    const unsigned long long s = block_inclusive_sum(c, warp_sums);
    if (threadIdx.x == blockDim.x - 1) tile_counts[blockIdx.x] = (uint32_t)s;
}

// one block of 1024 threads: offsets[t] = sum of tile_counts[0 .. t), offsets[tiles] = the total
__global__ void __launch_bounds__(1024) mock_scan_kernel(const uint32_t* tile_counts, uint64_t tiles, unsigned long long* offsets) {
    __shared__ unsigned long long warp_sums[32], round_total;
    unsigned long long carry = 0;
    for (uint64_t t0 = 0; t0 < tiles; t0 += blockDim.x) {
        const uint64_t t = t0 + threadIdx.x;
        const unsigned long long c = t < tiles ? tile_counts[t] : 0;
        const unsigned long long s = block_inclusive_sum(c, warp_sums);
        if (t < tiles) offsets[t] = carry + s - c;
        if (threadIdx.x == blockDim.x - 1) round_total = s;
        __syncthreads();
        carry += round_total;
        __syncthreads();
    }
    if (threadIdx.x == 0) offsets[tiles] = carry;
}

// tile b writes the indices of its set bits to out[offsets[b] ...], ascending; an index at position >= cap is not written
__global__ void __launch_bounds__(MOCK_THREADS) mock_scatter_kernel(const uint32_t* mask, uint64_t words, const unsigned long long* offsets,
                                                                    uint64_t cap, uint64_t* out) {
    __shared__ unsigned long long warp_sums[32];
    const unsigned long long tile_off = offsets[blockIdx.x];
    if (tile_off >= cap) return;  // uniform over the block: no thread reaches the scan below
    const uint64_t w0 = (uint64_t)blockIdx.x * MOCK_TILE_WORDS + (uint64_t)threadIdx.x * MOCK_WORDS_PER_THREAD;
    uint32_t m[MOCK_WORDS_PER_THREAD], c = 0;
    for (uint32_t w = 0; w < MOCK_WORDS_PER_THREAD; ++w) {
        m[w] = w0 + w < words ? mask[w0 + w] : 0;
        c += __popc(m[w]);
    }
    unsigned long long pos = tile_off + block_inclusive_sum(c, warp_sums) - c;
    for (uint32_t w = 0; w < MOCK_WORDS_PER_THREAD && pos < cap; ++w)
        for (uint32_t bits = m[w]; bits && pos < cap; bits &= bits - 1) out[pos++] = ((w0 + w) << 5) | (uint32_t)(__ffs(bits) - 1);
}

// Scratch of one check in ctx->stage_out, in this order: the pointer table (8 B per column) | bad flag (8 B) | mask
// (4 B per 32 flat indices) | tile counts (4 B per tile) | offsets (8 B per tile + 8) | the check's own (the lookup's slots).
struct MockScratch {
    uint64_t words, tiles;
    const Fr** ptrs;
    uint32_t *bad, *mask, *tile_counts;
    unsigned long long* offsets;
    char* extra;
};

static int32_t mock_scratch(b200zk_ctx* ctx, uint64_t total, uint64_t n_ptrs, size_t extra_bytes, MockScratch* s) {
    s->words = (total + 31) / 32;
    s->tiles = (s->words + MOCK_TILE_WORDS - 1) / MOCK_TILE_WORDS;
    const size_t o_bad = 8 * (size_t)n_ptrs, o_mask = o_bad + 8, o_cnt = o_mask + 4 * (size_t)((s->words + 1) & ~1ull);
    const size_t o_off = o_cnt + 4 * (size_t)((s->tiles + 1) & ~1ull), o_extra = o_off + 8 * (size_t)(s->tiles + 1);
    B2_TRY(scratch_reserve(ctx, ctx->stage_out, o_extra + extra_bytes));
    char* base = (char*)ctx->stage_out.p;
    s->ptrs = (const Fr**)base;
    s->bad = (uint32_t*)(base + o_bad);
    s->mask = (uint32_t*)(base + o_mask);
    s->tile_counts = (uint32_t*)(base + o_cnt);
    s->offsets = (unsigned long long*)(base + o_off);
    s->extra = base + o_extra;
    return B200ZK_OK;
}

static uint32_t mock_blocks(b200zk_ctx* ctx, uint64_t n) {
    uint64_t want = (n + MOCK_THREADS - 1) / MOCK_THREADS, cap = (uint64_t)ctx->sm_count * 16;
    if (want > cap) want = cap;
    return (uint32_t)(want ? want : 1);
}

// the mask written by a check -> *count_out = its set bits, rows_out[0 .. min(cap, count)) = their indices, ascending.
// rows_out in device memory is written in place; host memory receives the list through ctx->misc.
static int32_t mock_compact(b200zk_ctx* ctx, const MockScratch& s, uint64_t* rows_out, uint64_t cap, uint64_t* count_out) {
    uint64_t count = 0;
    if (s.tiles) {
        {
            ProfScope ps_(ctx, PROF_POLY);
            mock_count_kernel<<<(uint32_t)s.tiles, MOCK_THREADS, 0, ctx->stream>>>(s.mask, s.words, s.tile_counts);
            B2_LAUNCH_CHECK(ctx);
            mock_scan_kernel<<<1, 1024, 0, ctx->stream>>>(s.tile_counts, s.tiles, s.offsets);
            B2_LAUNCH_CHECK(ctx);
        }
        B2_TRY(d2h(ctx, &count, s.offsets + s.tiles, 8));
    }
    *count_out = count;
    const uint64_t take = count < cap ? count : cap;
    if (!take) return B200ZK_OK;
    uint64_t* dst = rows_out;
    const bool on_device = is_device_ptr(rows_out);
    if (!on_device) {
        B2_TRY(scratch_reserve(ctx, ctx->misc, 8 * (size_t)take));
        dst = (uint64_t*)ctx->misc.p;
    }
    {
        ProfScope ps_(ctx, PROF_POLY);
        mock_scatter_kernel<<<(uint32_t)s.tiles, MOCK_THREADS, 0, ctx->stream>>>(s.mask, s.words, s.offsets, take, dst);
        B2_LAUNCH_CHECK(ctx);
    }
    return on_device ? B200ZK_OK : d2h(ctx, rows_out, dst, 8 * (size_t)take);
}

static int32_t check_out(b200zk_ctx* ctx, const char* what, uint64_t* rows_out, uint64_t cap, uint64_t* count_out) {
    if (!count_out) return fail(ctx, B200ZK_E_INVALID, "%s: null count_out", what);
    if (cap && !rows_out) return fail(ctx, B200ZK_E_INVALID, "%s: null rows_out with cap = %llu", what, (unsigned long long)cap);
    return B200ZK_OK;
}

static int32_t check_columns(b200zk_ctx* ctx, const char* what, const char* name, const void* const* cols, uint32_t count) {
    if (!cols) return fail(ctx, B200ZK_E_INVALID, "%s: null %s table", what, name);
    for (uint32_t j = 0; j < count; ++j)
        if (!cols[j] || !is_device_ptr(cols[j])) return fail(ctx, B200ZK_E_INVALID, "%s: %s[%u] must be a device pointer", what, name, j);
    return B200ZK_OK;
}

int32_t nonzero_rows_run(b200zk_ctx* ctx, const Fr* values, uint64_t n, uint64_t* rows_out, uint64_t cap, uint64_t* count_out) {
    MockScratch s;
    B2_TRY(mock_scratch(ctx, n, 0, 0, &s));
    if (n) {
        ProfScope ps_(ctx, PROF_POLY);
        mock_nonzero_kernel<<<mock_blocks(ctx, n), MOCK_THREADS, 0, ctx->stream>>>(values, n, s.mask);
        B2_LAUNCH_CHECK(ctx);
    }
    return mock_compact(ctx, s, rows_out, cap, count_out);
}

int32_t lookup_missing_run(b200zk_ctx* ctx, const void* const* inputs, uint32_t n_inputs, const Fr* table, uint32_t k, uint64_t usable,
                           uint64_t* rows_out, uint64_t cap, uint64_t* count_out) {
    const uint64_t total = (uint64_t)n_inputs << k;
    const uint32_t log_slots = lk_log_slots(usable);
    MockScratch s;
    B2_TRY(mock_scratch(ctx, total, n_inputs, 4 * ((size_t)1 << log_slots), &s));
    uint32_t* slots = (uint32_t*)s.extra;
    B2_CUDA(ctx, cudaMemcpyAsync(s.ptrs, inputs, sizeof(void*) * n_inputs, cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(ctx, cudaMemsetAsync(slots, 0xFF, 4 * ((size_t)1 << log_slots), ctx->stream));
    {
        ProfScope ps_(ctx, PROF_POLY);
        B2_TRY(lookup_build_launch(ctx, table, usable, slots, log_slots));
        mock_lookup_miss_kernel<<<mock_blocks(ctx, total), MOCK_THREADS, 0, ctx->stream>>>(s.ptrs, k, total, table, usable, slots,
                                                                                           log_slots, s.mask);
        B2_LAUNCH_CHECK(ctx);
    }
    return mock_compact(ctx, s, rows_out, cap, count_out);
}

int32_t copy_check_run(b200zk_ctx* ctx, const void* const* cols, uint32_t n_cols, const uint64_t* next, uint32_t k, uint64_t* rows_out,
                       uint64_t cap, uint64_t* count_out) {
    const uint64_t total = (uint64_t)n_cols << k;
    MockScratch s;
    B2_TRY(mock_scratch(ctx, total, n_cols, 0, &s));
    B2_CUDA(ctx, cudaMemcpyAsync(s.ptrs, cols, sizeof(void*) * n_cols, cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(ctx, cudaMemsetAsync(s.bad, 0, 4, ctx->stream));
    {
        ProfScope ps_(ctx, PROF_POLY);
        mock_copy_kernel<<<mock_blocks(ctx, total), MOCK_THREADS, 0, ctx->stream>>>(s.ptrs, k, total, next, s.mask, s.bad);
        B2_LAUNCH_CHECK(ctx);
    }
    uint32_t bad = 0;
    B2_TRY(d2h(ctx, &bad, s.bad, 4));
    if (bad) return fail(ctx, B200ZK_E_INVALID, "copy_check: a next entry is >= n_cols * 2^k = %llu", (unsigned long long)total);
    return mock_compact(ctx, s, rows_out, cap, count_out);
}

}  // namespace b200zk

using namespace b200zk;

extern "C" {

int32_t b200zk_nonzero_rows(b200zk_ctx* ctx, const void* values_dev, uint64_t n, uint64_t* rows_out, uint64_t cap, uint64_t* count_out) {
    if (!ctx) return B200ZK_E_INVALID;
    B2_TRY(check_out(ctx, "nonzero_rows", rows_out, cap, count_out));
    Guard g(ctx);
    if (n && (!values_dev || !is_device_ptr(values_dev))) return fail(ctx, B200ZK_E_INVALID, "nonzero_rows: values must be a device pointer");
    return nonzero_rows_run(ctx, (const Fr*)values_dev, n, rows_out, cap, count_out);
}

int32_t b200zk_lookup_missing_rows(b200zk_ctx* ctx, const void* const* inputs_dev, uint32_t n_inputs, const void* table_dev, uint32_t k,
                                   uint64_t usable, uint64_t* rows_out, uint64_t cap, uint64_t* count_out) {
    if (!ctx) return B200ZK_E_INVALID;
    if (n_inputs < 1 || n_inputs > 64) return fail(ctx, B200ZK_E_INVALID, "lookup_missing_rows: n_inputs = %u (1 <= n_inputs <= 64)", n_inputs);
    if (k > 28) return fail(ctx, B200ZK_E_INVALID, "lookup_missing_rows: k = %u > 28", k);
    if (usable > (1ull << k))
        return fail(ctx, B200ZK_E_INVALID, "lookup_missing_rows: usable = %llu > 2^%u", (unsigned long long)usable, k);
    B2_TRY(check_out(ctx, "lookup_missing_rows", rows_out, cap, count_out));
    Guard g(ctx);
    B2_TRY(check_columns(ctx, "lookup_missing_rows", "inputs", inputs_dev, n_inputs));
    if (!table_dev || !is_device_ptr(table_dev)) return fail(ctx, B200ZK_E_INVALID, "lookup_missing_rows: table must be a device pointer");
    return lookup_missing_run(ctx, inputs_dev, n_inputs, (const Fr*)table_dev, k, usable, rows_out, cap, count_out);
}

int32_t b200zk_copy_check(b200zk_ctx* ctx, const void* const* cols_dev, uint32_t n_cols, const uint64_t* next_dev, uint32_t k,
                          uint64_t* rows_out, uint64_t cap, uint64_t* count_out) {
    if (!ctx) return B200ZK_E_INVALID;
    if (n_cols < 1) return fail(ctx, B200ZK_E_INVALID, "copy_check: n_cols = 0");
    if (k > 28) return fail(ctx, B200ZK_E_INVALID, "copy_check: k = %u > 28", k);
    B2_TRY(check_out(ctx, "copy_check", rows_out, cap, count_out));
    Guard g(ctx);
    B2_TRY(check_columns(ctx, "copy_check", "cols", cols_dev, n_cols));
    if (!next_dev || !is_device_ptr(next_dev)) return fail(ctx, B200ZK_E_INVALID, "copy_check: next must be a device pointer");
    return copy_check_run(ctx, cols_dev, n_cols, next_dev, k, rows_out, cap, count_out);
}

}  // extern "C"

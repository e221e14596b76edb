// The multiplicity column m(X) of the log-derivative lookup on the device: mv_lookup::Argument::prepare of
// halo2_proofs 1.1.0 @ scroll-tech/halo2 e5ddf67, where upstream builds a host index of the table and walks the inputs.
//
//   lookup_build_kernel    table rows -> an open-addressing set of row indices; a value's slot ends up holding the FIRST
//                          usable row with that value (the rule of the host mirror's index.emplace)
//   lookup_probe_kernel    every (input, row) finds its table row; counts are aggregated per warp before the atomic
//   lookup_finish_kernel   m[r] = count[r] in Montgomery form, zero on every other row
//
// The slot array only stores u32 row indices: a key is always read back from table[row], so the set costs 4 B per slot and
// the comparisons read the table, which stays in L2 for the hot values.  A slot, once claimed, only ever holds rows of one
// value (a thread only lowers it with atomicMin after comparing equal), so concurrent inserts of equal values meet in the
// same slot and the result does not depend on the schedule.
#include "lookup.cuh"

namespace b200zk {

__global__ void __launch_bounds__(256) lookup_build_kernel(const Fr* table, uint64_t usable, uint32_t* slots, uint32_t log_slots) {
    const uint64_t mask = (1ull << log_slots) - 1, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < usable; r += stride) {
        const LkKey key = lk_load(table + r);
        for (uint64_t h = lk_hash(key, log_slots);; h = (h + 1) & mask) {
            uint32_t cur = slots[h];
            if (cur == LK_EMPTY) {
                cur = atomicCAS(slots + h, LK_EMPTY, (uint32_t)r);
                if (cur == LK_EMPTY) break;  // claimed
            }
            if (lk_eq(lk_load(table + cur), key)) {
                // the slot only decreases: a row above the one already seen cannot win, so the many repeats of a padding
                // value skip the atomic on their shared slot
                if ((uint32_t)r < cur) atomicMin(slots + h, (uint32_t)r);
                break;
            }
        }
    }
}

// grid (x, n_inputs); whole warps walk the rows together so that __match_any_sync sees all 32 lanes
__global__ void __launch_bounds__(256) lookup_probe_kernel(const Fr* const* inputs, uint32_t k, const Fr* table, uint64_t usable,
                                                           const uint32_t* slots, uint32_t log_slots, unsigned long long* counts,
                                                           unsigned long long* missing) {
    const uint32_t j = blockIdx.y, lane = threadIdx.x & 31;
    const Fr* in = inputs[j];
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < usable; base += stride) {
        const uint64_t i = base + lane;
        const uint32_t row = i < usable ? lk_find(lk_load(in + i), table, slots, log_slots) : LK_EMPTY;
        const bool miss = i < usable && row == LK_EMPTY;
        // range-check inputs are dominated by a few values: one atomic per distinct row of the warp
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, row);
        if (row != LK_EMPTY && lane == (uint32_t)(__ffs(peers) - 1)) atomicAdd(counts + row, (unsigned long long)__popc(peers));
        if (miss) atomicMin(missing, (unsigned long long)(((uint64_t)j << k) | i));
    }
}

__global__ void __launch_bounds__(256) lookup_finish_kernel(const unsigned long long* counts, uint64_t usable, uint64_t n, Fr* m) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
        Fr v = Fr::zero();
        const uint64_t c = r < usable ? counts[r] : 0;
        if (c) {
            v.l.v[0] = (uint32_t)c;
            v.l.v[1] = (uint32_t)(c >> 32);
            v = v.to_mont();
        }
        uint4* q = reinterpret_cast<uint4*>(m + r);
        q[0] = make_uint4(v.l.v[0], v.l.v[1], v.l.v[2], v.l.v[3]);
        q[1] = make_uint4(v.l.v[4], v.l.v[5], v.l.v[6], v.l.v[7]);
    }
}

int32_t lookup_build_launch(b200zk_ctx* ctx, const Fr* table, uint64_t usable, uint32_t* slots, uint32_t log_slots) {
    if (!usable) return B200ZK_OK;
    lookup_build_kernel<<<lk_blocks(ctx, usable), 256, 0, ctx->stream>>>(table, usable, slots, log_slots);
    B2_LAUNCH_CHECK(ctx);
    return B200ZK_OK;
}

// scratch in ctx->stage_out: input pointer table | missing | counts (usable u64) | slots (>= 2 usable u32, a power of two)
int32_t lookup_multiplicities_run(b200zk_ctx* ctx, const void* const* inputs, uint32_t n_inputs, const Fr* table, uint32_t k,
                                  uint64_t usable, Fr* m_out, uint64_t* first_missing) {
    const uint64_t n = 1ull << k;
    const uint32_t log_slots = lk_log_slots(usable);
    const size_t o_ptr = 0, o_miss = 8 * 64, o_cnt = o_miss + 8, o_slot = o_cnt + 8 * (size_t)usable;
    const size_t total = o_slot + 4 * ((size_t)1 << log_slots);
    B2_TRY(scratch_reserve(ctx, ctx->stage_out, total));
    char* base = (char*)ctx->stage_out.p;
    auto* missing = (unsigned long long*)(base + o_miss);
    auto* counts = (unsigned long long*)(base + o_cnt);
    auto* slots = (uint32_t*)(base + o_slot);
    B2_CUDA(ctx, cudaMemcpyAsync(base + o_ptr, inputs, sizeof(void*) * n_inputs, cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(ctx, cudaMemsetAsync(missing, 0xFF, 8, ctx->stream));
    if (usable) B2_CUDA(ctx, cudaMemsetAsync(counts, 0, 8 * (size_t)usable, ctx->stream));
    B2_CUDA(ctx, cudaMemsetAsync(slots, 0xFF, 4 * ((size_t)1 << log_slots), ctx->stream));
    {
        ProfScope ps_(ctx, PROF_POLY);
        if (usable) {
            B2_TRY(lookup_build_launch(ctx, table, usable, slots, log_slots));
            uint32_t bx = lk_blocks(ctx, usable * n_inputs) / n_inputs;
            dim3 grid(bx ? bx : 1, n_inputs);
            lookup_probe_kernel<<<grid, 256, 0, ctx->stream>>>((const Fr* const*)(base + o_ptr), k, table, usable, slots, log_slots,
                                                               counts, missing);
            B2_LAUNCH_CHECK(ctx);
        }
        lookup_finish_kernel<<<lk_blocks(ctx, n), 256, 0, ctx->stream>>>(counts, usable, n, m_out);
        B2_LAUNCH_CHECK(ctx);
    }
    return d2h(ctx, first_missing, missing, 8);
}

}  // namespace b200zk

using namespace b200zk;

extern "C" {

int32_t b200zk_lookup_multiplicities(b200zk_ctx* ctx, const void* const* inputs_dev, uint32_t n_inputs, const void* table_dev,
                                     uint32_t k, uint64_t usable, void* m_out_dev, uint64_t* first_missing) {
    if (!ctx) return B200ZK_E_INVALID;
    if (n_inputs < 1 || n_inputs > 64) return fail(ctx, B200ZK_E_INVALID, "lookup_multiplicities: n_inputs = %u (1 <= n_inputs <= 64)", n_inputs);
    if (k > 28) return fail(ctx, B200ZK_E_INVALID, "lookup_multiplicities: k = %u > 28", k);
    if (usable > (1ull << k))
        return fail(ctx, B200ZK_E_INVALID, "lookup_multiplicities: usable = %llu > 2^%u", (unsigned long long)usable, k);
    if (!first_missing) return fail(ctx, B200ZK_E_INVALID, "lookup_multiplicities: null first_missing");
    if (!inputs_dev) return fail(ctx, B200ZK_E_INVALID, "lookup_multiplicities: null pointer table");
    Guard g(ctx);
    for (uint32_t j = 0; j < n_inputs; ++j)
        if (!inputs_dev[j] || !is_device_ptr(inputs_dev[j]))
            return fail(ctx, B200ZK_E_INVALID, "lookup_multiplicities: inputs[%u] must be a device pointer", j);
    if (!table_dev || !is_device_ptr(table_dev)) return fail(ctx, B200ZK_E_INVALID, "lookup_multiplicities: table must be a device pointer");
    if (!m_out_dev || !is_device_ptr(m_out_dev)) return fail(ctx, B200ZK_E_INVALID, "lookup_multiplicities: m_out must be a device pointer");
    return lookup_multiplicities_run(ctx, inputs_dev, n_inputs, (const Fr*)table_dev, k, usable, (Fr*)m_out_dev, first_missing);
}

}  // extern "C"

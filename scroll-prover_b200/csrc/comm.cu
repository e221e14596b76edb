// Multi-GPU side of libb200zk: the context-owned NCCL communicator and the point-range sharded MSM
// (SURVEY.md §8(b): "the ctx owns CUDA streams, NCCL comm, device pools"; §8(e): partition by point range,
// local Pippenger, all-gather of the per-rank partial points as raw bytes, G - 1 local additions).
//
// One process per GPU, one context per process; rank r of `world` computes  sum_{i in [lo_r, hi_r)} s_i * P_i  over
// its contiguous slice of the (replicated) SRS and the partial points (96 B each) are exchanged with ONE
// ncclAllGather on the context stream -- NCCL has no G1 reduction operator, and 96 B x world needs no custom kernel.
// The result is the same group element on every rank, normalised, so its bytes equal the single-GPU ones.
//
// NCCL is bound at run time (dlopen of libnccl.so.2: the copy the process already holds -- e.g. torch's -- is
// reused, and the library still loads on a machine without NCCL, where b200zk_ctx_comm_init fails loudly).
#include <dlfcn.h>
#include <nccl.h>

#include "common.cuh"
#include "ec.cuh"

namespace b200zk {

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    std::string err;
};

static NcclApi* nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* nm : names) {
            api.handle = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
        }
        if (!api.handle) {
            api.err = std::string("dlopen(libnccl.so.2) failed: ") + (dlerror() ? dlerror() : "?");
            return;
        }
        auto sym = [&](const char* s) -> void* {
            void* p = dlsym(api.handle, s);
            if (!p && api.err.empty()) api.err = std::string("NCCL symbol missing: ") + s;
            return p;
        };
        api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
        api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
        api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
    });
    return &api;
}

#define B2_NCCL(ctx, api, call)                                                                                       \
    do {                                                                                                              \
        ncclResult_t r__ = (call);                                                                                    \
        if (r__ != ncclSuccess)                                                                                       \
            return fail(ctx, B200ZK_E_CUDA, "%s failed: %s", #call, (api)->GetErrorString ? (api)->GetErrorString(r__) : "?"); \
    } while (0)

void shard_range(uint64_t n, int rank, int world, uint64_t* first, uint64_t* count) {
    // contiguous, sizes differ by at most one, the first (n mod world) ranks get the extra element
    uint64_t q = n / (uint64_t)world, r = n % (uint64_t)world, k = (uint64_t)rank;
    *first = k * q + (k < r ? k : r);
    *count = q + (k < r ? 1 : 0);
}

int32_t comm_destroy(b200zk_ctx* ctx) {
    if (ctx->nccl_comm) {
        NcclApi* api = nccl_api();
        if (api->CommDestroy) api->CommDestroy((ncclComm_t)ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    if (ctx->comm_buf) {
        cudaFree(ctx->comm_buf);
        ctx->comm_buf = nullptr;
    }
    ctx->comm_rank = 0;
    ctx->comm_world = 1;
    return B200ZK_OK;
}

}  // namespace b200zk

using namespace b200zk;

extern "C" {

int32_t b200zk_comm_unique_id(void* id128) {
    if (!id128) return B200ZK_E_INVALID;
    NcclApi* api = nccl_api();
    if (!api->GetUniqueId) return B200ZK_E_UNSUPPORTED;
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    if (api->GetUniqueId(&id) != ncclSuccess) return B200ZK_E_CUDA;
    memcpy(id128, &id, sizeof id);
    return B200ZK_OK;
}

int32_t b200zk_ctx_comm_init(b200zk_ctx* ctx, const void* id128, int rank, int world) {
    if (!ctx) return B200ZK_E_INVALID;
    if (world < 1 || rank < 0 || rank >= world) return fail(ctx, B200ZK_E_INVALID, "comm_init: rank %d of world %d", rank, world);
    Guard g(ctx);
    comm_destroy(ctx);
    if (world == 1) return B200ZK_OK;  // a single rank needs no communicator: the sharded entry points degenerate
    if (!id128) return fail(ctx, B200ZK_E_INVALID, "comm_init: null unique id");
    NcclApi* api = nccl_api();
    if (!api->CommInitRank || !api->AllGather) return fail(ctx, B200ZK_E_UNSUPPORTED, "comm_init: NCCL unavailable (%s)", api->err.c_str());
    ncclUniqueId id;
    memcpy(&id, id128, sizeof id);
    ncclComm_t comm = nullptr;
    B2_NCCL(ctx, api, api->CommInitRank(&comm, world, id, rank));
    ctx->nccl_comm = comm;
    ctx->comm_rank = rank;
    ctx->comm_world = world;
    B2_CUDA(ctx, cudaMalloc(&ctx->comm_buf, sizeof(Jacobian) * (size_t)(world + 1)));
    return B200ZK_OK;
}

int32_t b200zk_ctx_comm_info(const b200zk_ctx* ctx, int* rank, int* world) {
    if (!ctx) return B200ZK_E_INVALID;
    if (rank) *rank = ctx->comm_rank;
    if (world) *world = ctx->comm_world;
    return B200ZK_OK;
}

int32_t b200zk_shard_range(uint64_t n, int rank, int world, uint64_t* first, uint64_t* count) {
    if (world < 1 || rank < 0 || rank >= world || !first || !count) return B200ZK_E_INVALID;
    shard_range(n, rank, world, first, count);
    return B200ZK_OK;
}

int32_t b200zk_allgather_rows(b200zk_ctx* ctx, void* values_dev, uint32_t log_size) {
    if (!ctx) return B200ZK_E_INVALID;
    if (!values_dev || log_size > 30) return fail(ctx, B200ZK_E_INVALID, "allgather_rows: bad arguments");
    if (!is_device_ptr(values_dev)) return fail(ctx, B200ZK_E_INVALID, "allgather_rows: values must be device memory");
    Guard g(ctx);
    const uint64_t size = 1ull << log_size, world = (uint64_t)ctx->comm_world;
    if (world == 1) return B200ZK_OK;
    if (size % world) return fail(ctx, B200ZK_E_INVALID, "allgather_rows: world %llu does not divide 2^%u", (unsigned long long)world, log_size);
    NcclApi* api = nccl_api();
    const size_t bytes = sizeof(Fr) * (size / world);
    char* base = (char*)values_dev;
    // in place: the send buffer is this rank's slice inside the receive buffer
    B2_NCCL(ctx, api, api->AllGather(base + bytes * (size_t)ctx->comm_rank, base, bytes, ncclChar, (ncclComm_t)ctx->nccl_comm, ctx->stream));
    return B200ZK_OK;
}

// partial MSM over the SRS slice [first, first + n)
static int32_t msm_range_dev(b200zk_ctx* ctx, const b200zk_srs* srs, const void* scalars, uint64_t first, uint64_t n, Jacobian* res) {
    const void* sc_dev = nullptr;
    if (n) B2_TRY(stage_in(ctx, ctx->stage_in, scalars, sizeof(Fr) * n, &sc_dev));
    const Fr* sc = (const Fr*)sc_dev;
    return msm_srs(ctx, srs, first, &sc, 1, n, res);
}

int32_t b200zk_msm_g1_range(b200zk_ctx* ctx, const b200zk_srs* srs, const void* scalars, uint64_t first, uint64_t n, void* out_jacobian96) {
    if (!ctx) return B200ZK_E_INVALID;
    if (!srs || !out_jacobian96 || (n && !scalars)) return fail(ctx, B200ZK_E_INVALID, "msm_g1_range: null pointer");
    if (srs->ctx != ctx) return fail(ctx, B200ZK_E_INVALID, "msm_g1_range: SRS belongs to another context");
    if (first > srs->n || n > srs->n - first)
        return fail(ctx, B200ZK_E_INVALID, "msm_g1_range: [%llu, +%llu) exceeds the %llu bases", (unsigned long long)first,
                    (unsigned long long)n, (unsigned long long)srs->n);
    Guard g(ctx);
    return out_small(ctx, out_jacobian96, sizeof(Jacobian),
                     [&](void* res) { return msm_range_dev(ctx, srs, scalars, first, n, (Jacobian*)res); });
}

int32_t b200zk_msm_g1_sharded(b200zk_ctx* ctx, const b200zk_srs* srs, const void* scalars_slice, uint64_t n_total, void* out_jacobian96) {
    if (!ctx) return B200ZK_E_INVALID;
    if (!srs || !out_jacobian96) return fail(ctx, B200ZK_E_INVALID, "msm_g1_sharded: null pointer");
    if (srs->ctx != ctx) return fail(ctx, B200ZK_E_INVALID, "msm_g1_sharded: SRS belongs to another context");
    if (n_total > srs->n)
        return fail(ctx, B200ZK_E_INVALID, "msm_g1_sharded: %llu scalars but only %llu bases (assert_eq!(coeffs.len(), bases.len()))",
                    (unsigned long long)n_total, (unsigned long long)srs->n);
    uint64_t first, cnt;
    shard_range(n_total, ctx->comm_rank, ctx->comm_world, &first, &cnt);
    if (cnt && !scalars_slice) return fail(ctx, B200ZK_E_INVALID, "msm_g1_sharded: null scalar slice");
    Guard g(ctx);
    if (ctx->comm_world == 1)
        return out_small(ctx, out_jacobian96, sizeof(Jacobian),
                         [&](void* res) { return msm_range_dev(ctx, srs, scalars_slice, 0, n_total, (Jacobian*)res); });
    NcclApi* api = nccl_api();
    Jacobian* buf = (Jacobian*)ctx->comm_buf;  // [0 .. world) gathered partials, [world] this rank's partial / the sum
    Jacobian* mine = buf + ctx->comm_world;
    B2_TRY(msm_range_dev(ctx, srs, scalars_slice, first, cnt, mine));
    B2_NCCL(ctx, api, api->AllGather(mine, buf, sizeof(Jacobian), ncclChar, (ncclComm_t)ctx->nccl_comm, ctx->stream));
    B2_TRY(g1_sum_run(ctx, buf, (uint64_t)ctx->comm_world, mine));
    return deliver(ctx, out_jacobian96, mine, sizeof(Jacobian));
}

}  // extern "C"

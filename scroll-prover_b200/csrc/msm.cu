// BN254 G1 multi-scalar multiplication (Pippenger bucket method) for sm_90a.
//
// Device replacement for halo2_proofs::arithmetic::best_multiexp / multiexp_serial and therefore
// ParamsKZG::commit / commit_lagrange (halo2_proofs/src/arithmetic.rs, src/poly/kzg/commitment.rs @
// scroll-tech/halo2 e5ddf67, pin /root/reference/Cargo.lock:1886-1888; reached from
// /root/reference/integration/src/prove.rs:37-39).  The result is the same group element
// sum_i s_i * P_i, returned normalised, so its bytes equal the reference's `to_affine()` output.
//
// Pipeline (DESIGN.md "MSM"); all of it on the context stream, no host synchronisation inside:
//   1 msm_count       scalar -> canonical (one Montgomery product), signed c-bit digits -> digits[w*n+i]; digits per
//                     coarse bin (256 buckets) counted in shared memory
//   2 scan            exclusive prefix sum of the bin counts (three kernels)
//   3 msm_partition + msm_bin_sort (+ msm_big_* for giant bins)   two-level counting sort of (table index | sign) into
//                     bucket order: tiles ordered by bin in shared memory and written as runs, then every bin ordered by
//                     its fine key; no global atomic per digit
//   4 msm_accumulate  lock-step segmented reduction: every thread owns L consecutive sorted entries and adds affine
//                     bases into an XYZZ accumulator (8M+2S per add); buckets wholly inside a chunk are stored
//                     directly, the <= 2 cut runs become partial records
//   5 msm_combine_*   partial records: ordinary buckets by their head record, GIANT buckets (> 4L entries: millions
//                     of equal digits in real witness columns) by a log-depth level reduction
//   6 msm_rowcol_sums + msm_bit_sums   sum_b b*B_b per bucket set with a short critical path (row / column sums, then
//                     bit-sliced weighted sums: independent subset sums instead of a dependent suffix scan)
//   7 msm_finish      one block per column: Horner over the bit sums and the bucket sets, normalisation to (x, y, 1)
// With a precomputed SRS (tables 2^(c*w) P_i, built at registration) all windows share ONE bucket set.
// BATCHES: up to 32 columns over the same bases run through one pipeline (bucket set = column * Ws + window; the grids of
// count / partition carry the column in blockIdx.y), so the fixed phases are paid once per batch (msm_run_batch).
// Zero scalars and zero digits are skipped (witness columns are mostly zeros / small values).
#include "common.cuh"
#include "ec.cuh"

namespace b200zk {

static constexpr uint32_t PART_INVALID = 0x1fffffffu;  // also the bucket-id mask
static constexpr uint32_t PART_GIANT = 0x20000000u;
static constexpr uint32_t PART_STARTS = 0x80000000u;
static constexpr uint32_t PART_ENDS = 0x40000000u;
static constexpr int MSM_MAX_BATCH = 32;
static constexpr int ACC_L_DEFAULT = 256;  // sorted entries per accumulate thread (B200ZK_ACC_L overrides, experiments)

struct MsmPlan {
    uint32_t c, W, B;   // window bits, windows, buckets per window (2^(c-1))
    uint32_t Ws;        // bucket sets per column: W, or 1 when the SRS holds precomputed 2^(c*w) multiples of every base
    uint32_t batch;     // columns (scalar vectors over the SAME bases) summed in one pipeline; bucket set = col * Ws + w
    uint64_t stride;    // precomputed SRS: table w starts at bases + w*stride (0 otherwise)
    uint64_t NB;        // batch * Ws * B
};

// Batched MSM: up to MSM_MAX_BATCH columns over the same bases go through ONE count / sort / accumulate / reduce pipeline
// (their bucket sets lie side by side), so the latency-bound phases -- scans, the bucket reduction, the final Horner --
// are paid once per batch instead of once per column.  This is what the hundreds of 2^20-row columns of the inner
// (zkEVM super-circuit) proof need; a 2^24+ column fills the machine alone and runs with batch = 1.
struct MsmCols {
    const Fr* p[MSM_MAX_BATCH];
};

__device__ __forceinline__ void ld_affine(const Affine* p, Fq& x, Fq& y) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
    x.l.v[0] = a.x; x.l.v[1] = a.y; x.l.v[2] = a.z; x.l.v[3] = a.w;
    x.l.v[4] = b.x; x.l.v[5] = b.y; x.l.v[6] = b.z; x.l.v[7] = b.w;
    y.l.v[0] = c.x; y.l.v[1] = c.y; y.l.v[2] = c.z; y.l.v[3] = c.w;
    y.l.v[4] = d.x; y.l.v[5] = d.y; y.l.v[6] = d.z; y.l.v[7] = d.w;
}

// ---- bucket sort: a two-level counting sort with no global atomic per digit ----------------------------------------
// A bucket b of set s has the global id s*B + b.  Its COARSE BIN is b >> FB: K = B >> FB bins per set of F = 2^FB buckets
// each (FB = min(8, c - 1), so that the FINE key b & (F - 1) is one byte).  Bin id = s*K + b>>FB, hence bucket id = bin*F +
// fine, and bins in id order are buckets in id order.
//   msm_count      recode every scalar once -> digits[w*n + i]; count digits per bin in shared memory, one global add per
//                  (block, bin)
//   scan           exclusive prefix sum of the bin counts -> bin_off (and bin_cur, the partition's cursors)
//   msm_partition  a block takes a tile of one window's digits, counts its bins in shared memory, reserves one contiguous
//                  run per bin (one global add per (tile, bin)), orders the tile by bin in shared memory and writes entry +
//                  fine key linearly into the runs.  Concurrent blocks reserve neighbouring runs, so L2 merges the run ends
//   msm_bin_sort   one block per bin: counting sort by the fine key, SORT_CH entries at a time ordered in shared memory,
//                  writes the bin's F offsets and its entries in bucket order
//   msm_big_*      bins above SORT_BIG entries (a giant bucket: millions of equal digits) are split over a whole grid instead
static constexpr int SORT_T = 512;                              // threads per block of the sort kernels
static constexpr int PART_T = 512, PART_ITEMS = 16, PART_TILE = PART_T * PART_ITEMS;  // digits per partition block
static constexpr uint32_t PART_STAGE_K = 8192;                  // up to this many bins a tile is ordered in shared memory
static constexpr int SORT_CH = 4096;                            // entries msm_bin_sort orders in shared memory at a time
static constexpr uint32_t SORT_FB_MAX = 8;                      // fine key = one byte
static constexpr uint32_t SORT_BIG = 1u << 17;                  // larger bins take the multi-block path
static constexpr uint32_t COUNT_LOCAL_MAX = 28672;              // bins counted in one block's shared memory (112 KiB)

struct SortPlan {
    uint32_t FB, K;      // fine bits, bins per bucket set
    uint32_t wpg;        // windows per msm_count group (plain bases; the precomputed SRS has one set and one group)
};

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// shared-memory add with one atomic per warp when every active lane has the same key (a giant bucket of a skewed witness
// column puts whole warps on one counter); otherwise one atomic per lane (__match_any_sync grouping costs more than the
// conflicts it saves on spread keys).  Every lane of the warp must call it.  Returns the old value + this lane's rank.
__device__ __forceinline__ uint32_t agg_add(uint32_t* ctr, uint32_t key, bool active) {
    const uint32_t act = __ballot_sync(0xffffffffu, active);
    const uint32_t kmin = __reduce_min_sync(0xffffffffu, active ? key : 0xffffffffu);
    const uint32_t kmax = __reduce_max_sync(0xffffffffu, active ? key : 0u);
    if (act && kmin == kmax) {
        const uint32_t lane = lane_id(), leader = __ffs(act) - 1;
        uint32_t base = 0;
        if (lane == leader) base = atomicAdd(&ctr[kmin], (uint32_t)__popc(act));
        base = __shfl_sync(0xffffffffu, base, leader);
        return base + __popc(act & ((1u << lane) - 1));
    }
    return active ? atomicAdd(&ctr[key], 1u) : 0u;
}

// grid = (blocks, column, window group).  Every scalar once: canonical form, signed digits -> digits[w*n + i]
// (magnitude | sign<<31, 0 = skip) for the windows of this group; bin counts in shared memory, flushed with one global
// add per (block, bin).
__global__ void __launch_bounds__(SORT_T) msm_count(MsmCols cols, uint64_t n, MsmPlan pl, SortPlan sp, uint32_t* __restrict__ bin_cnt,
                                                   uint32_t* __restrict__ digits_all) {
    extern __shared__ uint32_t lc[];
    const uint32_t col = blockIdx.y;
    const Fr* scalars = cols.p[0];
#pragma unroll
    for (int q = 1; q < MSM_MAX_BATCH; ++q)
        if (q == (int)col) scalars = cols.p[q];  // no dynamic indexing of kernel parameters
    const uint32_t wlo = blockIdx.z * sp.wpg, whi = min(pl.W, wlo + sp.wpg);
    const uint32_t nloc = (pl.Ws == 1 ? 1u : whi - wlo) * sp.K;
    for (uint32_t b = threadIdx.x; b < nloc; b += blockDim.x) lc[b] = 0;
    __syncthreads();
    uint32_t* digits = digits_all + (uint64_t)col * pl.W * n;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x; i0 < n; i0 += stride) {  // i0 is block-uniform: whole warps iterate
        const uint64_t i = i0 + threadIdx.x;
        const bool ok = i < n;
        uint32_t l[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (ok) {
            Fr s = scalars[i];
            if (!s.is_zero()) {
                s = s.from_mont();
#pragma unroll
                for (int k = 0; k < 8; ++k) l[k] = s.l.v[k];
            }
        }
        const uint32_t c = pl.c, mask = (1u << c) - 1, half = 1u << (c - 1);
        uint32_t carry = 0;
        for (uint32_t w = 0; w < whi; ++w) {
            uint32_t v = (l[0] & mask) + carry;
#pragma unroll
            for (int k = 0; k < 7; ++k) l[k] = __funnelshift_r(l[k], l[k + 1], c);
            l[7] >>= c;
            uint32_t enc;
            if (v > half) {
                enc = (1u << c) - v;  // magnitude of the negative digit (0 when v == 2^c)
                carry = 1;
                if (enc) enc |= 0x80000000u;
            } else {
                enc = v;
                carry = 0;
            }
            if (w < wlo) continue;
            if (ok) digits[(uint64_t)w * n + i] = enc;
            const uint32_t bin = ((enc & 0x7fffffffu) - 1) >> sp.FB;
            agg_add(lc, (pl.Ws == 1 ? 0u : (w - wlo) * sp.K) + bin, enc != 0);
        }
    }
    __syncthreads();
    uint32_t* gc = bin_cnt + ((uint64_t)col * pl.Ws + (pl.Ws == 1 ? 0u : wlo)) * sp.K;
    for (uint32_t b = threadIdx.x; b < nloc; b += blockDim.x)
        if (lc[b]) atomicAdd(&gc[b], lc[b]);
}

// block-wide exclusive scan of ctr[0..K) in place (PART_T threads); returns the total
__device__ __forceinline__ uint32_t part_block_scan(uint32_t* ctr, uint32_t K, uint32_t* wsum) {
    const uint32_t per = (K + PART_T - 1) / PART_T, lo = threadIdx.x * per, lane = lane_id(), warp = threadIdx.x >> 5;
    uint32_t s = 0;
    for (uint32_t k = 0; k < per; ++k)
        if (lo + k < K) s += ctr[lo + k];
    uint32_t x = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= (uint32_t)o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t v = lane < PART_T / 32 ? wsum[lane] : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= (uint32_t)o) v += y;
        }
        if (lane < PART_T / 32) wsum[lane] = v;  // inclusive over warps
    }
    __syncthreads();
    uint32_t run = (warp ? wsum[warp - 1] : 0u) + x - s;
    const uint32_t total = wsum[PART_T / 32 - 1];
    for (uint32_t k = 0; k < per; ++k)
        if (lo + k < K) {
            const uint32_t v = ctr[lo + k];
            ctr[lo + k] = run;
            run += v;
        }
    __syncthreads();
    return total;
}

// grid = (tiles of PART_TILE digits, col * W + w): stage the tile's entries by bin.  staged[pos] = (i + w*stride) | sign,
// fine[pos] = bucket & (F - 1), with pos inside the run this block reserved in its bin (one global add per (tile, bin)).
// With K <= PART_STAGE_K the tile is first ordered by bin in shared memory, so that a warp's stores fall into a few runs
// instead of 32 scattered sectors; wider windows write each entry straight into its run.
__global__ void __launch_bounds__(PART_T) msm_partition(const uint32_t* __restrict__ digits, uint64_t n, MsmPlan pl, SortPlan sp,
                                                       uint32_t* __restrict__ bin_cur, uint32_t* __restrict__ staged,
                                                       uint8_t* __restrict__ fine) {
    extern __shared__ uint32_t lc[];
    __shared__ uint32_t wsum[PART_T / 32];
    const uint32_t cw = blockIdx.y;
    const uint32_t col = cw / pl.W, w = cw - col * pl.W;
    const uint32_t* dg = digits + (uint64_t)cw * n;
    uint32_t* cur = bin_cur + ((uint64_t)col * pl.Ws + (pl.Ws == 1 ? 0u : w)) * sp.K;
    const uint32_t woff = (uint32_t)((uint64_t)w * pl.stride);
    const uint32_t K = sp.K, fmask = (1u << sp.FB) - 1;
    for (uint32_t b = threadIdx.x; b < K; b += blockDim.x) lc[b] = 0;
    const uint64_t i0 = (uint64_t)blockIdx.x * PART_TILE + threadIdx.x;
    uint32_t d[PART_ITEMS];
#pragma unroll
    for (int k = 0; k < PART_ITEMS; ++k) {
        const uint64_t i = i0 + (uint64_t)k * PART_T;
        d[k] = i < n ? dg[i] : 0u;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PART_ITEMS; ++k) agg_add(lc, ((d[k] & 0x7fffffffu) - 1) >> sp.FB, d[k] != 0);
    __syncthreads();
    if (K > PART_STAGE_K) {
        for (uint32_t b = threadIdx.x; b < K; b += blockDim.x)
            if (lc[b]) lc[b] = atomicAdd(&cur[b], lc[b]);
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PART_ITEMS; ++k) {
            const uint32_t bk = (d[k] & 0x7fffffffu) - 1;
            const uint32_t pos = agg_add(lc, bk >> sp.FB, d[k] != 0);
            if (d[k]) {
                staged[pos] = ((uint32_t)(i0 + (uint64_t)k * PART_T) + woff) | (d[k] & 0x80000000u);
                fine[pos] = (uint8_t)(bk & fmask);
            }
        }
        return;
    }
    uint32_t* gd = lc + K;           // global run start - local run start, per bin
    uint32_t* se = gd + K;           // the tile's entries ordered by bin
    uint32_t* sk = se + PART_TILE;   // bin << 8 | fine key
#pragma unroll 4
    for (uint32_t b = threadIdx.x; b < K; b += blockDim.x) gd[b] = lc[b] ? atomicAdd(&cur[b], lc[b]) : 0u;
    __syncthreads();
    const uint32_t total = part_block_scan(lc, K, wsum);
    for (uint32_t b = threadIdx.x; b < K; b += blockDim.x) gd[b] -= lc[b];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PART_ITEMS; ++k) {
        const uint32_t bk = (d[k] & 0x7fffffffu) - 1;
        const uint32_t p = agg_add(lc, bk >> sp.FB, d[k] != 0);
        if (d[k]) {
            se[p] = ((uint32_t)(i0 + (uint64_t)k * PART_T) + woff) | (d[k] & 0x80000000u);
            sk[p] = (bk >> sp.FB) << 8 | (bk & fmask);
        }
    }
    __syncthreads();
    for (uint32_t t = threadIdx.x; t < total; t += blockDim.x) {
        const uint32_t key = sk[t], dst = gd[key >> 8] + t;
        staged[dst] = se[t];
        fine[dst] = (uint8_t)(key & 0xffu);
    }
}

// exclusive scan of the F <= 256 counters in ctr[] (in place) by warp 0; returns nothing, the caller syncs
__device__ __forceinline__ void fine_exclusive_scan(uint32_t* ctr, uint32_t F) {
    if (threadIdx.x >= 32) return;
    const uint32_t lane = lane_id(), per = (F + 31) / 32, lo = lane * per;
    uint32_t v[8], s = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        v[k] = (k < (int)per && lo + k < F) ? ctr[lo + k] : 0u;
        s += v[k];
    }
    uint32_t x = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= (uint32_t)o) x += y;
    }
    uint32_t run = x - s;
#pragma unroll
    for (int k = 0; k < 8; ++k)
        if (k < (int)per && lo + k < F) {
            ctr[lo + k] = run;
            run += v[k];
        }
}

__device__ __forceinline__ void bin_range(const uint32_t* bin_off, uint64_t nbins, const uint32_t* total, uint64_t sb,
                                          uint32_t& start, uint32_t& end) {
    start = bin_off[sb];
    end = sb + 1 < nbins ? bin_off[sb + 1] : *total;
}

// one block per bin: counting sort by the fine key, offsets[bin*F + f] and the bin's sorted entries.  A bin above SORT_BIG
// entries is only listed (big_list[0] = count, then bin ids) for the multi-block kernels.
__global__ void __launch_bounds__(SORT_T, 3) msm_bin_sort(const uint32_t* __restrict__ bin_off, uint64_t nbins, SortPlan sp,
                                                      const uint32_t* __restrict__ staged, const uint8_t* __restrict__ fine,
                                                      uint32_t* __restrict__ offsets, uint32_t* __restrict__ entries,
                                                      uint32_t* __restrict__ big_list) {
    __shared__ uint32_t ctr[1u << SORT_FB_MAX], lc[1u << SORT_FB_MAX], cnt[1u << SORT_FB_MAX], gd[1u << SORT_FB_MAX];
    __shared__ uint32_t se[SORT_CH];
    __shared__ uint8_t sf[SORT_CH];
    const uint64_t sb = blockIdx.x;
    const uint32_t F = 1u << sp.FB;
    uint32_t start, end;
    bin_range(bin_off, nbins, offsets + nbins * F, sb, start, end);
    if (end - start > SORT_BIG) {
        if (threadIdx.x == 0) big_list[1 + atomicAdd(big_list, 1u)] = (uint32_t)sb;
        return;
    }
    for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) ctr[f] = 0;
    __syncthreads();
    for (uint32_t p0 = start; p0 < end; p0 += SORT_CH) {  // SORT_CH / SORT_T independent loads in flight per thread
        uint32_t fk[SORT_CH / SORT_T];
#pragma unroll
        for (int k = 0; k < SORT_CH / SORT_T; ++k) {
            const uint32_t p = p0 + k * SORT_T + threadIdx.x;
            fk[k] = p < end ? fine[p] : 0u;
        }
#pragma unroll
        for (int k = 0; k < SORT_CH / SORT_T; ++k) agg_add(ctr, fk[k], p0 + k * SORT_T + threadIdx.x < end);
    }
    __syncthreads();
    fine_exclusive_scan(ctr, F);
    __syncthreads();
    for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) {
        ctr[f] += start;
        offsets[sb * F + f] = ctr[f];
    }
    // SORT_CH entries at a time: order the chunk by fine key in shared memory, then write it out linearly, so that a
    // warp's stores fall into a few bucket runs
    for (uint32_t c0 = start; c0 < end; c0 += SORT_CH) {
        const uint32_t len = end - c0 < (uint32_t)SORT_CH ? end - c0 : (uint32_t)SORT_CH;
        for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) lc[f] = 0;
        __syncthreads();
        uint32_t e[SORT_CH / SORT_T], fk[SORT_CH / SORT_T];
#pragma unroll
        for (int k = 0; k < SORT_CH / SORT_T; ++k) {
            const uint32_t t = k * SORT_T + threadIdx.x;
            e[k] = t < len ? staged[c0 + t] : 0u;
            fk[k] = t < len ? fine[c0 + t] : 0u;
        }
#pragma unroll
        for (int k = 0; k < SORT_CH / SORT_T; ++k) agg_add(lc, fk[k], k * SORT_T + threadIdx.x < len);
        __syncthreads();
        for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) cnt[f] = lc[f];
        __syncthreads();
        fine_exclusive_scan(lc, F);
        __syncthreads();
        for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) {
            gd[f] = ctr[f] - lc[f];
            ctr[f] += cnt[f];
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < SORT_CH / SORT_T; ++k) {
            const bool ok = k * SORT_T + threadIdx.x < len;
            const uint32_t p = agg_add(lc, fk[k], ok);
            if (ok) {
                se[p] = e[k];
                sf[p] = (uint8_t)fk[k];
            }
        }
        __syncthreads();
        for (uint32_t t = threadIdx.x; t < len; t += blockDim.x) entries[gd[sf[t]] + t] = se[t];
        __syncthreads();
    }
}

// big bins, pass 1: every block of the grid counts its slice of each listed bin; one global add per (block, bucket)
__global__ void __launch_bounds__(SORT_T) msm_big_count(const uint32_t* __restrict__ bin_off, uint64_t nbins, SortPlan sp,
                                                       const uint8_t* __restrict__ fine, const uint32_t* __restrict__ offsets,
                                                       const uint32_t* __restrict__ big_list, uint32_t* __restrict__ big_cnt) {
    __shared__ uint32_t ctr[1u << SORT_FB_MAX];
    const uint32_t F = 1u << sp.FB, nbig = big_list[0];
    for (uint32_t j = 0; j < nbig; ++j) {
        uint32_t start, end;
        bin_range(bin_off, nbins, offsets + nbins * F, big_list[1 + j], start, end);
        const uint32_t lo = start + (uint32_t)((uint64_t)(end - start) * blockIdx.x / gridDim.x);
        const uint32_t hi = start + (uint32_t)((uint64_t)(end - start) * (blockIdx.x + 1) / gridDim.x);
        for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) ctr[f] = 0;
        __syncthreads();
        for (uint32_t p0 = lo; p0 < hi; p0 += SORT_T) {
            const uint32_t p = p0 + threadIdx.x;
            agg_add(ctr, p < hi ? fine[p] : 0u, p < hi);
        }
        __syncthreads();
        for (uint32_t f = threadIdx.x; f < F; f += blockDim.x)
            if (ctr[f]) atomicAdd(&big_cnt[(uint64_t)j * 2 * F + f], ctr[f]);
        __syncthreads();
    }
}

// big bins, pass 2: bucket bases from the pass-1 totals; each block reserves its run per bucket (one global add per
// (block, bucket) on the cursor beside the totals) and scatters its slice into it
__global__ void __launch_bounds__(SORT_T, 1) msm_big_scatter(const uint32_t* __restrict__ bin_off, uint64_t nbins, SortPlan sp,
                                                         const uint32_t* __restrict__ staged, const uint8_t* __restrict__ fine,
                                                         uint32_t* __restrict__ offsets, uint32_t* __restrict__ entries,
                                                         const uint32_t* __restrict__ big_list, uint32_t* __restrict__ big_cnt) {
    __shared__ uint32_t base[1u << SORT_FB_MAX], ctr[1u << SORT_FB_MAX];
    const uint32_t F = 1u << sp.FB, nbig = big_list[0];
    for (uint32_t j = 0; j < nbig; ++j) {
        const uint32_t sb = big_list[1 + j];
        uint32_t start, end;
        bin_range(bin_off, nbins, offsets + nbins * F, sb, start, end);
        const uint32_t lo = start + (uint32_t)((uint64_t)(end - start) * blockIdx.x / gridDim.x);
        const uint32_t hi = start + (uint32_t)((uint64_t)(end - start) * (blockIdx.x + 1) / gridDim.x);
        uint32_t* tot = big_cnt + (uint64_t)j * 2 * F;
        for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) {
            base[f] = tot[f];
            ctr[f] = 0;
        }
        __syncthreads();
        for (uint32_t p0 = lo; p0 < hi; p0 += SORT_T) {
            const uint32_t p = p0 + threadIdx.x;
            agg_add(ctr, p < hi ? fine[p] : 0u, p < hi);
        }
        fine_exclusive_scan(base, F);
        __syncthreads();
        for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) {
            if (blockIdx.x == 0) offsets[(uint64_t)sb * F + f] = start + base[f];
            if (ctr[f]) ctr[f] = start + base[f] + atomicAdd(&tot[F + f], ctr[f]);
        }
        __syncthreads();
        for (uint32_t p0 = lo; p0 < hi; p0 += SORT_T) {
            const uint32_t p = p0 + threadIdx.x;
            const bool ok = p < hi;
            const uint32_t e = ok ? staged[p] : 0u;
            const uint32_t pos = agg_add(ctr, ok ? fine[p] : 0u, ok);
            if (ok) entries[pos] = e;
        }
        __syncthreads();
    }
}

// ---- exclusive scan of uint32 counts (three kernels) -----------------------------------------
static constexpr int SCAN_TPB = 256, SCAN_ITEMS = 16, SCAN_TILE = SCAN_TPB * SCAN_ITEMS;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* total) {
    __shared__ uint32_t warp_sums[SCAN_TPB / 32];
    uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= (uint32_t)o) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint32_t s = (lane < SCAN_TPB / 32) ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= (uint32_t)o) s += y;
        }
        if (lane < SCAN_TPB / 32) warp_sums[lane] = s;  // inclusive over warps
    }
    __syncthreads();
    uint32_t warp_off = wid ? warp_sums[wid - 1] : 0;
    *total = warp_sums[SCAN_TPB / 32 - 1];
    uint32_t r = warp_off + x - v;
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(SCAN_TPB) scan_tile_sums(const uint32_t* in, uint64_t n, uint32_t* tile_sums) {
    uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_ITEMS;
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k)
        if (base + k < n) s += in[base + k];
    uint32_t total;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
// one block: exclusive scan of the tile sums in chunks of SCAN_TPB with a running carry
__global__ void __launch_bounds__(SCAN_TPB) scan_tile_offsets(uint32_t* tile_sums, uint32_t ntiles, uint32_t* grand_total,
                                                              unsigned long long* running) {
    uint32_t carry = 0;
    for (uint32_t base = 0; base < ntiles; base += SCAN_TPB) {
        uint32_t i = base + threadIdx.x;
        uint32_t v = i < ntiles ? tile_sums[i] : 0, total;
        uint32_t ex = block_exclusive_scan(v, &total);
        if (i < ntiles) tile_sums[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) {
        *grand_total = carry;
        if (running) atomicAdd(running, (unsigned long long)carry);
    }
}
__global__ void __launch_bounds__(SCAN_TPB) scan_apply(const uint32_t* in, uint64_t n, const uint32_t* tile_offs, uint32_t* out,
                                                     uint32_t* out2) {
    uint64_t base = (uint64_t)blockIdx.x * SCAN_TILE + (uint64_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        v[k] = (base + k < n) ? in[base + k] : 0;
        s += v[k];
    }
    uint32_t total;
    uint32_t off = block_exclusive_scan(s, &total) + tile_offs[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        if (base + k < n) {
            out[base + k] = off;
            out2[base + k] = off;
        }
        off += v[k];
    }
}

// ---- bucket accumulation ------------------------------------------------------------------------
__device__ __forceinline__ void st_xyzz(XYZZ* p, const XYZZ& v) {
    uint4* q = reinterpret_cast<uint4*>(p);
    const Fq* f = &v.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        q[2 * k] = make_uint4(f[k].l.v[0], f[k].l.v[1], f[k].l.v[2], f[k].l.v[3]);
        q[2 * k + 1] = make_uint4(f[k].l.v[4], f[k].l.v[5], f[k].l.v[6], f[k].l.v[7]);
    }
}
__device__ __forceinline__ XYZZ ld_xyzz(const XYZZ* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    XYZZ v;
    Fq* f = &v.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        uint4 a = q[2 * k], b = q[2 * k + 1];
        f[k].l.v[0] = a.x; f[k].l.v[1] = a.y; f[k].l.v[2] = a.z; f[k].l.v[3] = a.w;
        f[k].l.v[4] = b.x; f[k].l.v[5] = b.y; f[k].l.v[6] = b.z; f[k].l.v[7] = b.w;
    }
    return v;
}

// offsets has NB + 1 entries (offsets[NB] = M sorted entries).  Perfect load balance: thread tau sums exactly the
// sorted entries [tau*L, (tau+1)*L) in lock step with its warp (one mixed add per iteration for every lane).
// Buckets that lie wholly inside the range are stored directly; the (at most two) runs cut by the range ends are
// emitted as partial records.  Records of ordinary buckets are merged by msm_combine_heads (a bucket of <= BIG
// entries is cut into <= BIG/L + 1 pieces); records of GIANT buckets (millions of equal digits in real witness
// columns) go through the log-depth msm_combine_level reduction instead.
__global__ void __launch_bounds__(256, 2)
msm_accumulate(const Affine* __restrict__ bases, const uint32_t* __restrict__ entries, const uint32_t* __restrict__ offsets,
               uint64_t NB, XYZZ* __restrict__ buckets, uint32_t* __restrict__ part_id, XYZZ* __restrict__ part_val,
               uint64_t nthreads, uint32_t* __restrict__ giant_flag, uint32_t ACC_L) {
    uint64_t tau = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tau >= nthreads) return;
    const uint32_t M = offsets[NB];
    const uint32_t BIG_BUCKET = 4 * ACC_L;  // buckets above this size are split over threads
    uint64_t start = tau * ACC_L;
    part_id[2 * tau] = PART_INVALID;
    part_id[2 * tau + 1] = PART_INVALID;
    if (start >= M) return;
    uint32_t end = (start + ACC_L < M) ? (uint32_t)(start + ACC_L) : M;
    uint64_t lo = 0, hi = NB;  // largest b with offsets[b] <= start
    while (hi - lo > 1) {
        uint64_t mid = (lo + hi) >> 1;
        if (offsets[mid] <= start) lo = mid; else hi = mid;
    }
    uint32_t b = (uint32_t)lo;
    uint32_t bucket_start = offsets[b], bucket_end = offsets[b + 1];
    bool run_starts = (bucket_start == (uint32_t)start);
    uint32_t slot = 0;
    XYZZ acc = XYZZ::identity();
    uint32_t pos = (uint32_t)start;
    while (true) {
        bool at_end = (pos == end);
        if (at_end || pos == bucket_end) {
            bool run_ends = (pos == bucket_end);
            if (run_starts && run_ends) {
                st_xyzz(buckets + b, acc);
            } else {
                uint32_t giant = (bucket_end - bucket_start > BIG_BUCKET) ? PART_GIANT : 0u;
                if (giant) *giant_flag = 1u;  // benign race: every writer stores the same value
                part_id[2 * tau + slot] = b | giant | (run_starts ? PART_STARTS : 0u) | (run_ends ? PART_ENDS : 0u);
                st_xyzz(part_val + 2 * tau + slot, acc);
                ++slot;
            }
            if (at_end) break;
            acc = XYZZ::identity();
            bucket_start = pos;
            do { ++b; bucket_end = offsets[b + 1]; } while (bucket_end == pos);  // skip empty buckets
            run_starts = true;
        }
        uint32_t e = entries[pos];
        Fq px, py;
        ld_affine(bases + (e & 0x7fffffffu), px, py);
        if (!(px.is_zero() && py.is_zero())) {
            if (e & 0x80000000u) py = py.neg();
            xyzz_madd(acc, px, py);
        }
        ++pos;
    }
}

// ordinary (non-giant) buckets: the head record sums the few following records up to the one that ends the bucket
__global__ void __launch_bounds__(128) msm_combine_heads(const uint32_t* __restrict__ part_id, const XYZZ* __restrict__ part_val,
                                                         uint64_t nrec, XYZZ* __restrict__ buckets) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrec) return;
    uint32_t id = part_id[r];
    if ((id & PART_INVALID) == PART_INVALID || (id & PART_GIANT) || !(id & PART_STARTS)) return;
    XYZZ sum = ld_xyzz(part_val + r);
    uint64_t k = r;
    while (!(id & PART_ENDS)) {
        ++k;
        if (k >= nrec) break;
        id = part_id[k];
        if ((id & PART_INVALID) == PART_INVALID) { id = 0; continue; }
        XYZZ v = ld_xyzz(part_val + k);
        xyzz_add(sum, v);
    }
    st_xyzz(buckets + (part_id[r] & PART_INVALID), sum);
}

// One level of the GIANT-bucket reduction: thread sigma scans LR consecutive records (sorted by bucket; invalid and,
// on the first level, non-giant records are skipped), sums runs of equal bucket id; a run that saw both the STARTS
// and the ENDS record is complete and is stored, otherwise it is re-emitted (<= 2 per thread) for the next level.
static constexpr int COMBINE_LR = 64;
__global__ void __launch_bounds__(128) msm_combine_level(const uint32_t* __restrict__ in_id, const XYZZ* __restrict__ in_val,
                                                         uint64_t nrec, XYZZ* __restrict__ buckets, uint32_t* __restrict__ out_id,
                                                         XYZZ* __restrict__ out_val, uint64_t nthreads,
                                                         const uint32_t* __restrict__ giant_flag) {
    if (*giant_flag == 0) return;  // no giant bucket in this MSM (the common case): nothing to reduce
    uint64_t sigma = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (sigma >= nthreads) return;
    out_id[2 * sigma] = PART_INVALID;
    out_id[2 * sigma + 1] = PART_INVALID;
    uint64_t r0 = sigma * COMBINE_LR, r1 = r0 + COMBINE_LR;
    if (r1 > nrec) r1 = nrec;
    bool have = false;
    uint32_t cur = 0, flags = 0, slot = 0;
    XYZZ acc = XYZZ::identity();
    auto flush = [&]() {
        if (!have) return;
        if ((flags & PART_STARTS) && (flags & PART_ENDS)) {
            st_xyzz(buckets + cur, acc);
        } else {
            out_id[2 * sigma + slot] = cur | flags | PART_GIANT;
            st_xyzz(out_val + 2 * sigma + slot, acc);
            ++slot;
        }
    };
    for (uint64_t r = r0; r < r1; ++r) {
        uint32_t id = in_id[r];
        if ((id & PART_INVALID) == PART_INVALID || !(id & PART_GIANT)) continue;
        uint32_t bkt = id & PART_INVALID;
        if (!have || bkt != cur) {
            flush();
            have = true;
            cur = bkt;
            flags = id & (PART_STARTS | PART_ENDS);
            acc = ld_xyzz(in_val + r);
        } else {
            flags |= id & (PART_STARTS | PART_ENDS);
            XYZZ v = ld_xyzz(in_val + r);
            xyzz_add(acc, v);
        }
    }
    flush();
}

// last level (few records): the head record of every giant bucket sums forward to the record that ends it
__global__ void __launch_bounds__(128) msm_combine_final(const uint32_t* __restrict__ part_id, const XYZZ* __restrict__ part_val,
                                                         uint64_t nrec, XYZZ* __restrict__ buckets, const uint32_t* __restrict__ giant_flag) {
    if (*giant_flag == 0) return;
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrec) return;
    uint32_t id = part_id[r];
    if ((id & PART_INVALID) == PART_INVALID || !(id & PART_GIANT) || !(id & PART_STARTS)) return;
    XYZZ sum = ld_xyzz(part_val + r);
    uint64_t k = r;
    while (!(id & PART_ENDS)) {
        ++k;
        if (k >= nrec) break;
        id = part_id[k];
        if ((id & PART_INVALID) == PART_INVALID || !(id & PART_GIANT)) { id = 0; continue; }
        XYZZ v = ld_xyzz(part_val + k);
        xyzz_add(sum, v);
    }
    st_xyzz(buckets + (part_id[r] & PART_INVALID), sum);
}

// ---- bucket reduction ---------------------------------------------------------------------------
// S = sum_{i<B} (i+1) B_i for every bucket set, with a SHORT critical path (the old running-sum + doubling tree had
// ~100 dependent point additions and ~200 dependent doublings; this has ~40 additions and kc doublings):
// view the set as a matrix i = hi*2^kc + lo;  Row_hi = sum_lo B, Col_lo = sum_hi B   (block tree sums), then
//   S = WS(Col) + 2^kc * WS(Row) + sum(Row),     WS(V) = sum_j j V_j = sum_{j>=1} Suffix_j(V)   (parallel suffix scan).
static constexpr int RED_T = 128;   // 4 blocks/SM at 128 registers: the sums are latency-bound, more blocks in flight win

// block tree sum through shared memory (result valid in thread 0).  A register-shuffle version (32 x SHFL.DOWN per level and
// lane, one shared-memory hand-over between the warps) does more work: every lane of a shuffle level executes the
// 14-multiplication addition (31 of 32 results are discarded at the last level) and the extra live XYZZ pushes the kernels
// into spills at 128 registers.
__device__ __forceinline__ void block_tree_sum(XYZZ& v, XYZZ* sh) {  // result valid in thread 0
    st_xyzz(sh + threadIdx.x, v);
    __syncthreads();
    for (uint32_t s = blockDim.x >> 1; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            XYZZ a = ld_xyzz(sh + threadIdx.x), b = ld_xyzz(sh + threadIdx.x + s);
            xyzz_add(a, b);
            st_xyzz(sh + threadIdx.x, a);
        }
        __syncthreads();
    }
    v = ld_xyzz(sh);
}

// grid = (rows + cols, Ws); block j < rows sums row j, block rows + j sums column j.  vec[set][0..rows) | [rows..rows+cols)
__global__ void __launch_bounds__(RED_T, 4) msm_rowcol_sums(const XYZZ* __restrict__ buckets, uint32_t B, uint32_t kc, XYZZ* __restrict__ vec) {
    __shared__ XYZZ sh[RED_T];
    const uint32_t cols = 1u << kc, rows = B >> kc;
    const XYZZ* bk = buckets + (uint64_t)blockIdx.y * B;
    XYZZ acc = XYZZ::identity();
    if (blockIdx.x < rows) {
        const XYZZ* r = bk + (uint64_t)blockIdx.x * cols;
        for (uint32_t lo = threadIdx.x; lo < cols; lo += blockDim.x) {
            XYZZ v = ld_xyzz(r + lo);
            xyzz_add(acc, v);
        }
    } else {
        uint32_t lo = blockIdx.x - rows;
        for (uint32_t hi = threadIdx.x; hi < rows; hi += blockDim.x) {
            XYZZ v = ld_xyzz(bk + (uint64_t)hi * cols + lo);
            xyzz_add(acc, v);
        }
    }
    block_tree_sum(acc, sh);
    if (threadIdx.x == 0) st_xyzz(vec + (uint64_t)blockIdx.y * (rows + cols) + blockIdx.x, acc);
}

// WS(V) = sum_j j V_j over a vector of m = 2^q elements, BIT-SLICED:  WS = sum_{b<q} 2^b S_b,  S_b = sum_{j: bit b of j} V_j.
// The q subset sums are independent block tree sums (depth ~ m/(2*RED_T) + log2 RED_T additions instead of the ~90 dependent
// additions of a suffix scan); msm_finish folds them with q - 1 doublings.
// grid = (q_max + 1, 2, sets): blockIdx.y = 0 the Row vector (m = rows), 1 the Col vector (m = cols); blockIdx.x = bit b, and
// blockIdx.x == q_max of the Row vector computes its plain total sum(Row).  out[set][which][b], stride (q_max + 1).
__global__ void __launch_bounds__(RED_T, 4) msm_bit_sums(const XYZZ* __restrict__ vec, uint32_t B, uint32_t kc, uint32_t q_max,
                                                         XYZZ* __restrict__ out) {
    __shared__ XYZZ sh[RED_T];
    const uint32_t cols = 1u << kc, rows = B >> kc;
    const uint32_t which = blockIdx.y, b = blockIdx.x;
    const uint32_t m = which == 0 ? rows : cols;
    const XYZZ* v = vec + (uint64_t)blockIdx.z * (rows + cols) + (which == 0 ? 0 : rows);
    XYZZ acc = XYZZ::identity();
    const bool total = (b == q_max);
    if (total ? (which == 0) : ((1u << b) < m)) {
        for (uint32_t j = threadIdx.x; j < m; j += blockDim.x)
            if (total || ((j >> b) & 1u)) {
                XYZZ e = ld_xyzz(v + j);
                xyzz_add(acc, e);
            }
    }
    block_tree_sum(acc, sh);
    if (threadIdx.x == 0) st_xyzz(out + ((uint64_t)blockIdx.z * 2 + which) * (q_max + 1) + b, acc);
}

// one block per column of the batch: warp 0 folds the Row bit sums, warp 1 the Col bit sums (Horner with doublings), then
// thread 0 combines  S = WS(Col) + 2^kc WS(Row) + sum(Row)  per bucket set, the window Horner, and normalises.
__global__ void __launch_bounds__(64) msm_finish(MsmPlan pl, uint32_t kc, uint32_t q_max, const XYZZ* __restrict__ bits_all, Jacobian* out_all) {
    __shared__ XYZZ ws[2];
    const uint32_t cols = 1u << kc, rows = pl.B >> kc;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    Jacobian* out = out_all + blockIdx.x;
    XYZZ acc = XYZZ::identity();
    for (uint32_t w = pl.Ws; w-- > 0;) {
        const uint64_t set = (uint64_t)blockIdx.x * pl.Ws + w;
        const XYZZ* bits = bits_all + set * 2 * (q_max + 1);
        if (lane == 0) {
            const uint32_t m = warp == 0 ? rows : cols;
            const XYZZ* bv = bits + (uint64_t)warp * (q_max + 1);
            XYZZ h = XYZZ::identity();
            uint32_t q = 0;
            while ((1u << q) < m) ++q;
            for (uint32_t b = q; b-- > 0;) {
                if (!h.is_identity()) h = xyzz_dbl(h);
                XYZZ e = ld_xyzz(bv + b);
                xyzz_add(h, e);
            }
            st_xyzz(ws + warp, h);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (!acc.is_identity())                                    // (always the identity when Ws == 1: skip the c doublings)
                for (uint32_t d = 0; d < pl.c; ++d) acc = xyzz_dbl(acc);
            XYZZ s = ld_xyzz(ws);                                      // WS(Row)
            for (uint32_t d = 0; d < kc; ++d) s = xyzz_dbl(s);
            XYZZ t = ld_xyzz(bits + q_max), u = ld_xyzz(ws + 1);       // sum(Row), WS(Col)
            xyzz_add(s, t);
            xyzz_add(s, u);
            xyzz_add(acc, s);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = xyzz_to_jacobian_normalized(acc);
}

// ---- small helpers exposed through the ABI --------------------------------------------------------
__global__ void g1_sum_kernel(const Jacobian* pts, uint64_t count, Jacobian* out) {
    if (threadIdx.x || blockIdx.x) return;
    XYZZ acc = XYZZ::identity();
    for (uint64_t i = 0; i < count; ++i) {
        XYZZ p = xyzz_from_jacobian(pts[i]);
        xyzz_add(acc, p);
    }
    *out = xyzz_to_jacobian_normalized(acc);
}

__global__ void __launch_bounds__(128) g1_generator_mul_kernel(const Fr* scalars, uint64_t n, Affine* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr s = scalars[i].from_mont();
    Fq gx = Fq::one(), gy = Fq::one().dbl();  // generator (1, 2)
    XYZZ acc = XYZZ::identity();
    for (int limb = 7; limb >= 0; --limb)
        for (int b = 31; b >= 0; --b) {
            acc = xyzz_dbl(acc);
            if ((s.l.v[limb] >> b) & 1) xyzz_madd(acc, gx, gy);
        }
    out[i] = xyzz_to_affine(acc);
}

// ---------------------------------------------------------------------------------------------
static uint32_t pick_window(uint64_t n) {
    if (n < 32) return n < 4 ? 2 : 4;
    double best = 1e300;
    uint32_t bc = 8;
    for (uint32_t c = 5; c <= 23; ++c) {
        uint32_t W = 254 / c + 1;
        if ((double)n * W >= 4.0e9) continue;  // sorted-entry positions are 32-bit
        double cost = (double)n * W * 10.0 + (double)W * (double)(1ull << c) * 40.0 + (double)W * 4096.0;
        if (cost < best) {
            best = cost;
            bc = c;
        }
    }
    return bc;
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// out[i] = 2^c * in[i] (affine): one table of the precomputed SRS from the previous one
__global__ void __launch_bounds__(128) srs_shift_kernel(const Affine* __restrict__ in, Affine* __restrict__ out, uint64_t n, uint32_t c) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Affine a = in[i];
    XYZZ p = xyzz_from_affine(a);
    for (uint32_t d = 0; d < c; ++d) p = xyzz_dbl(p);
    out[i] = xyzz_to_affine(p);
}

static uint32_t pick_window_precomputed(uint64_t n) {
    double best = 1e300;
    uint32_t bc = 10;
    for (uint32_t c = 8; c <= 23; ++c) {
        uint32_t W = 254 / c + 1;
        if ((double)n * W >= 2.0e9) continue;  // entry = table index (31 bits) | sign
        // 10 MODMUL per bucket addition; ~40 MODMUL-equivalents per bucket slot for the (latency-bound) reduction
        // (the ratio of the reduction's time per bucket to the accumulation's time per addition)
        double cost = (double)n * W * 10.0 + (double)(1ull << c) * 40.0;
        if (cost < best) {
            best = cost;
            bc = c;
        }
    }
    return bc;
}

// tables[w] = 2^(c*w) * bases, w = 0..W-1, laid out back to back (stride n); tables[0] must already hold the bases
static int32_t srs_precompute_run(b200zk_ctx* ctx, Affine* tables, uint64_t n, uint32_t c, uint32_t W) {
    for (uint32_t w = 1; w < W; ++w) {
        srs_shift_kernel<<<(uint32_t)((n + 127) / 128), 128, 0, ctx->stream>>>(tables + (uint64_t)(w - 1) * n, tables + (uint64_t)w * n, n, c);
        B2_LAUNCH_CHECK(ctx);
    }
    return B200ZK_OK;
}

// how many columns of n scalars one batched pipeline may take (sorted-entry positions are 32-bit; scratch stays ~2 GiB)
static uint32_t msm_max_batch(uint64_t n, uint32_t pre_c) {
    uint32_t c = pre_c ? pre_c : pick_window(n);
    uint64_t per_col = (n ? n : 1) * (254 / c + 1);
    uint64_t b = (1ull << 28) / per_col;
    return (uint32_t)(b < 1 ? 1 : (b > MSM_MAX_BATCH ? MSM_MAX_BATCH : b));
}

// pre_c != 0: `bases` is a precomputed SRS (W tables of stride pre_stride) built for window pre_c.
// cols[0 .. batch): device pointers of `batch` scalar vectors of n elements each; out_dev[0 .. batch).
static int32_t msm_run_batch(b200zk_ctx* ctx, const Affine* bases, const Fr* const* cols, uint32_t batch, uint64_t n, Jacobian* out_dev,
                             uint32_t pre_c, uint64_t pre_stride) {
    if (n >= (1ull << 31)) return fail(ctx, B200ZK_E_UNSUPPORTED, "msm: n = %llu >= 2^31", (unsigned long long)n);
    if (batch < 1 || batch > (uint32_t)MSM_MAX_BATCH) return fail(ctx, B200ZK_E_INVALID, "msm: batch %u out of range [1,%d]", batch, MSM_MAX_BATCH);
    MsmPlan pl;
    pl.c = pre_c ? pre_c : (ctx->msm_window ? ctx->msm_window : pick_window(n));
    if (pl.c < 2 || pl.c > 24) return fail(ctx, B200ZK_E_INVALID, "msm: window %u out of range [2,24]", pl.c);
    pl.W = 254 / pl.c + 1;
    pl.B = 1u << (pl.c - 1);
    pl.Ws = pre_c ? 1 : pl.W;
    pl.batch = batch;
    pl.stride = pre_c ? pre_stride : 0;
    pl.NB = (uint64_t)batch * pl.Ws * pl.B;
    uint64_t max_entries = n * pl.W * batch;
    if (max_entries >= 0xffffffffull) return fail(ctx, B200ZK_E_UNSUPPORTED, "msm: n*W*batch too large for window %u", pl.c);
    MsmCols colp;
    for (int q = 0; q < MSM_MAX_BATCH; ++q) colp.p[q] = cols[q < (int)batch ? q : 0];
    ctx->last_c = pl.c;
    ctx->last_windows = pl.W;
    ctx->last_adds = n * pl.W;

    const uint32_t ACC_L = ctx->msm_acc_l ? ctx->msm_acc_l : (uint32_t)ACC_L_DEFAULT;
    uint64_t nthreads = (max_entries + ACC_L - 1) / ACC_L;
    if (nthreads == 0) nthreads = 1;
    SortPlan sp;
    sp.FB = pl.c - 1 < SORT_FB_MAX ? pl.c - 1 : SORT_FB_MAX;
    sp.K = pl.B >> sp.FB;
    sp.wpg = pl.Ws == 1 ? pl.W : (COUNT_LOCAL_MAX / sp.K < 1 ? 1 : (COUNT_LOCAL_MAX / sp.K < pl.W ? COUNT_LOCAL_MAX / sp.K : pl.W));
    const uint32_t groups = (pl.W + sp.wpg - 1) / sp.wpg;
    const uint64_t nbins = pl.NB >> sp.FB;
    const uint32_t F = 1u << sp.FB;
    const uint64_t max_big = max_entries / SORT_BIG + 1;
    uint32_t ntiles = (uint32_t)((nbins + SCAN_TILE - 1) / SCAN_TILE);
    // carve the scratch arena.  Sort scratch beyond O(NB): digits and entries (4 B per slot each) and the one-byte fine keys,
    // which share the accumulate's partial records (idle until the sort is done; >= 1 B per slot at the default ACC_L)
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    size_t o_offs = carve(4 * (pl.NB + 1));
    size_t o_bcnt = carve(4 * (nbins + 1)), o_boff = carve(4 * (nbins + 1)), o_bcur = carve(4 * (nbins + 1));
    size_t o_big = carve(4 * (max_big + 1)), o_bigc = carve(4 * 2 * F * max_big);
    size_t o_tiles = carve(4 * (size_t)(ntiles + 1));
    size_t o_flag = carve(256);
    size_t o_entries = carve(4 * (max_entries + 4));
    size_t o_digits = carve(4 * (max_entries + 4));
    size_t o_buckets = carve(sizeof(XYZZ) * pl.NB);
    size_t pval_bytes = sizeof(XYZZ) * 2 * nthreads;
    size_t o_pid = carve(4 * 2 * nthreads), o_pval = carve(pval_bytes > max_entries + 16 ? pval_bytes : max_entries + 16);
    uint64_t nthreads2 = (2 * nthreads + COMBINE_LR - 1) / COMBINE_LR;
    size_t o_pid2 = carve(4 * 2 * nthreads2), o_pval2 = carve(sizeof(XYZZ) * 2 * nthreads2);
    const uint32_t kc = pl.c / 2;                       // columns = 2^kc, rows = B / 2^kc  (c - 1 = kc + kr)
    const uint32_t red_cols = 1u << kc, red_rows = pl.B >> kc;
    const uint32_t sets = batch * pl.Ws;
    size_t red_len = (size_t)sets * (red_rows + red_cols);
    uint32_t q_max = 0;  // bits of the longer of the Row / Col vectors
    while ((1u << q_max) < (red_rows > red_cols ? red_rows : red_cols)) ++q_max;
    size_t o_gr = carve(sizeof(XYZZ) * red_len), o_sums = carve(sizeof(XYZZ) * 2 * (q_max + 1) * sets);
    B2_TRY(scratch_reserve(ctx, ctx->msm_work, off));
    char* base = (char*)ctx->msm_work.p;
    uint32_t* offsets = (uint32_t*)(base + o_offs);
    uint32_t* bin_cnt = (uint32_t*)(base + o_bcnt);
    uint32_t* bin_off = (uint32_t*)(base + o_boff);
    uint32_t* bin_cur = (uint32_t*)(base + o_bcur);
    uint32_t* big_list = (uint32_t*)(base + o_big);
    uint32_t* big_cnt = (uint32_t*)(base + o_bigc);
    uint32_t* tiles = (uint32_t*)(base + o_tiles);
    uint32_t* giant_flag = (uint32_t*)(base + o_flag);
    uint32_t* staged = (uint32_t*)(base + o_entries);  // partitioned entries; the sorted ones go to the dead digits
    uint32_t* digits = (uint32_t*)(base + o_digits);
    uint32_t* entries = digits;
    uint32_t* pid2 = (uint32_t*)(base + o_pid2);
    XYZZ* pval2 = (XYZZ*)(base + o_pval2);
    XYZZ* buckets = (XYZZ*)(base + o_buckets);
    uint32_t* pid = (uint32_t*)(base + o_pid);
    XYZZ* pval = (XYZZ*)(base + o_pval);
    uint8_t* fine = (uint8_t*)(base + o_pval);
    XYZZ* grpR = (XYZZ*)(base + o_gr);
    XYZZ* red_sums = (XYZZ*)(base + o_sums);

    cudaStream_t st = ctx->stream;
    B2_CUDA(ctx, cudaMemsetAsync(bin_cnt, 0, 4 * (nbins + 1), st));
    B2_CUDA(ctx, cudaMemsetAsync(big_list, 0, o_tiles - o_big, st));  // list count and the big bins' totals / cursors
    B2_CUDA(ctx, cudaMemsetAsync(giant_flag, 0, 4, st));
    B2_CUDA(ctx, cudaMemsetAsync(buckets, 0, sizeof(XYZZ) * pl.NB, st));
    const size_t count_smem = 4ull * (pl.Ws == 1 ? 1u : sp.wpg) * sp.K;
    const size_t part_smem = sp.K > PART_STAGE_K ? 4ull * sp.K : 4ull * (2 * sp.K + 2 * PART_TILE);
    if (!(ctx->smem_optin & (1u << 9))) {
        // the largest request: K = 2^15 bins of a window of 24 bits (msm_count takes one window per group there)
        const int most = (int)(4 * (1u << (24 - 1 - SORT_FB_MAX)));
        B2_CUDA(ctx, cudaFuncSetAttribute(msm_count, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
        B2_CUDA(ctx, cudaFuncSetAttribute(msm_partition, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
        ctx->smem_optin |= 1u << 9;
    }
    if (n) {
        // one wave of resident blocks (as many per SM as the bin counters allow); each flushes its counters once
        int per_sm = 1;
        B2_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, msm_count, SORT_T, count_smem));
        if (per_sm < 1) per_sm = 1;
        uint64_t want = (n + SORT_T - 1) / SORT_T;
        uint32_t per = ((uint32_t)ctx->sm_count * (uint32_t)per_sm + batch * groups - 1) / (batch * groups);
        uint32_t blocks = (uint32_t)(want < per ? want : per);
        {
            ProfScope ps_(ctx, PROF_MSM_COUNT);
            msm_count<<<dim3(blocks, batch, groups), SORT_T, count_smem, st>>>(colp, n, pl, sp, bin_cnt, digits);
        }
        B2_LAUNCH_CHECK(ctx);
    }
    {
        ProfScope ps_(ctx, PROF_MSM_SCAN);
        scan_tile_sums<<<ntiles, SCAN_TPB, 0, st>>>(bin_cnt, nbins, tiles);
        B2_LAUNCH_CHECK(ctx);
        scan_tile_offsets<<<1, SCAN_TPB, 0, st>>>(tiles, ntiles, offsets + pl.NB, ctx->msm_adds_dev);
        B2_LAUNCH_CHECK(ctx);
        scan_apply<<<ntiles, SCAN_TPB, 0, st>>>(bin_cnt, nbins, tiles, bin_off, bin_cur);
        B2_LAUNCH_CHECK(ctx);
    }
    if (n) {
        {
            ProfScope ps_(ctx, PROF_MSM_SCATTER);
            // grid.y = col * W + w, issued window-major (x fastest): concurrent blocks reserve neighbouring runs of one window
            uint32_t pblocks = (uint32_t)((n + PART_TILE - 1) / PART_TILE);
            msm_partition<<<dim3(pblocks, batch * pl.W), PART_T, part_smem, st>>>(digits, n, pl, sp, bin_cur, staged, fine);
            B2_LAUNCH_CHECK(ctx);
            msm_bin_sort<<<(uint32_t)nbins, SORT_T, 0, st>>>(bin_off, nbins, sp, staged, fine, offsets, entries, big_list);
            B2_LAUNCH_CHECK(ctx);
            uint32_t gblocks = (uint32_t)ctx->sm_count * 2;
            msm_big_count<<<gblocks, SORT_T, 0, st>>>(bin_off, nbins, sp, fine, offsets, big_list, big_cnt);
            B2_LAUNCH_CHECK(ctx);
            msm_big_scatter<<<gblocks, SORT_T, 0, st>>>(bin_off, nbins, sp, staged, fine, offsets, entries, big_list, big_cnt);
        }
        B2_LAUNCH_CHECK(ctx);
        uint32_t ablocks = (uint32_t)((nthreads + 255) / 256);
        {
            ProfScope ps_(ctx, PROF_MSM_ACCUM);
            msm_accumulate<<<ablocks, 256, 0, st>>>(bases, entries, offsets, pl.NB, buckets, pid, pval, nthreads, giant_flag, ACC_L);
        }
        B2_LAUNCH_CHECK(ctx);
        {
            ProfScope ps_(ctx, PROF_MSM_COMBINE);
            uint64_t nrec = 2 * nthreads;
            msm_combine_heads<<<(uint32_t)((nrec + 127) / 128), 128, 0, st>>>(pid, pval, nrec, buckets);
            B2_LAUNCH_CHECK(ctx);
            uint32_t *in_id = pid, *out_id = pid2;
            XYZZ *in_val = pval, *out_val = pval2;
            while (nrec > 2048) {
                uint64_t nt = (nrec + COMBINE_LR - 1) / COMBINE_LR;
                msm_combine_level<<<(uint32_t)((nt + 127) / 128), 128, 0, st>>>(in_id, in_val, nrec, buckets, out_id, out_val, nt, giant_flag);
                B2_LAUNCH_CHECK(ctx);
                nrec = 2 * nt;
                uint32_t* ti = in_id; in_id = out_id; out_id = ti;
                XYZZ* tv = in_val; in_val = out_val; out_val = tv;
            }
            msm_combine_final<<<(uint32_t)((nrec + 127) / 128), 128, 0, st>>>(in_id, in_val, nrec, buckets, giant_flag);
            B2_LAUNCH_CHECK(ctx);
        }
    }
    {
        ProfScope ps_(ctx, PROF_MSM_REDUCE);
        msm_rowcol_sums<<<dim3(red_rows + red_cols, sets), RED_T, 0, st>>>(buckets, pl.B, kc, grpR);
        B2_LAUNCH_CHECK(ctx);
        msm_bit_sums<<<dim3(q_max + 1, 2, sets), RED_T, 0, st>>>(grpR, pl.B, kc, q_max, red_sums);
        B2_LAUNCH_CHECK(ctx);
        msm_finish<<<batch, 64, 0, st>>>(pl, kc, q_max, red_sums, out_dev);
        B2_LAUNCH_CHECK(ctx);
    }
    return B200ZK_OK;
}

int32_t msm_bases(b200zk_ctx* ctx, const Affine* bases, const Fr* scalars, uint64_t n, Jacobian* out_dev) {
    return msm_run_batch(ctx, bases, &scalars, 1, n, out_dev, 0, 0);
}

// ---- the SRS handle's device side: this file alone reads dev_bases, pre_c and pre_W ---------------------------------
int32_t srs_init(b200zk_ctx* ctx, b200zk_srs* s, const void* g1_affine) {
    const uint64_t n = s->n;
    s->dev_bases = nullptr;
    s->pre_c = 0;
    s->pre_W = 1;
    size_t bytes = sizeof(Affine) * (n ? n : 1);
    if (ctx->srs_precompute && n >= (1ull << 16)) {
        // keep 2^(c*w) * P_i for every window w: all windows then share ONE bucket set (no per-window reduction, no
        // Horner doublings) and a wider window pays off.  Costs W x the base storage; skipped when memory is short.
        uint32_t c = pick_window_precomputed(n), W = 254 / c + 1;
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && (double)bytes * W < 0.35 * (double)free_b) {
            s->pre_c = c;
            s->pre_W = W;
            bytes *= W;
        }
    }
    cudaError_t e = cudaMalloc(&s->dev_bases, bytes);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        s->dev_bases = nullptr;
        return fail(ctx, B200ZK_E_OOM, "srs_register: cudaMalloc(%zu) failed", bytes);
    }
    cudaMemcpyKind kind = is_device_ptr(g1_affine) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    e = n ? cudaMemcpyAsync(s->dev_bases, g1_affine, sizeof(Affine) * n, kind, ctx->stream) : cudaSuccess;
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        srs_free(s);
        return fail(ctx, B200ZK_E_CUDA, "srs_register: upload failed: %s", cudaGetErrorString(e));
    }
    if (s->pre_c) {
        int32_t rc = srs_precompute_run(ctx, (Affine*)s->dev_bases, n, s->pre_c, s->pre_W);
        if (rc == B200ZK_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = B200ZK_E_CUDA;
        if (rc != B200ZK_OK) {
            srs_free(s);
            return fail(ctx, rc, "srs_register: precomputation failed");
        }
    }
    return B200ZK_OK;
}

void srs_free(b200zk_srs* s) {
    if (s->dev_bases) cudaFree(s->dev_bases);
    s->dev_bases = nullptr;
}

// a commit over a short prefix of a large precomputed SRS is cheaper with the plain bases (table 0) and a window sized for n
// than with the handle's wide window (2^(c-1) buckets to reduce)
static uint32_t srs_pre_c(const b200zk_srs* s, uint64_t n) { return (s->pre_c && n * 16 >= s->n) ? s->pre_c : 0; }

uint32_t msm_srs_max_batch(const b200zk_srs* s, uint64_t n) { return msm_max_batch(n, srs_pre_c(s, n)); }

int32_t msm_srs(b200zk_ctx* ctx, const b200zk_srs* s, uint64_t first, const Fr* const* cols, uint32_t count, uint64_t n,
                Jacobian* out_dev) {
    const uint32_t pre_c = srs_pre_c(s, n), bmax = msm_max_batch(n, pre_c);
    // the precomputed tables 2^(c*w) P_i lie at stride s->n: a slice of them is the same layout with an offset
    const Affine* bases = (const Affine*)s->dev_bases + first;
    for (uint32_t j = 0; j < count; j += bmax)
        B2_TRY(msm_run_batch(ctx, bases, cols + j, count - j < bmax ? count - j : bmax, n, out_dev + j, pre_c, s->n));
    return B200ZK_OK;
}

int32_t g1_sum_run(b200zk_ctx* ctx, const Jacobian* pts, uint64_t count, Jacobian* out_dev) {
    g1_sum_kernel<<<1, 32, 0, ctx->stream>>>(pts, count, out_dev);
    B2_LAUNCH_CHECK(ctx);
    return B200ZK_OK;
}

int32_t g1_generator_mul_run(b200zk_ctx* ctx, const Fr* scalars, uint64_t n, Affine* out) {
    if (!n) return B200ZK_OK;
    g1_generator_mul_kernel<<<(uint32_t)((n + 127) / 128), 128, 0, ctx->stream>>>(scalars, n, out);
    B2_LAUNCH_CHECK(ctx);
    return B200ZK_OK;
}

}  // namespace b200zk

"""numpy model of the device MSM's bucket sort (csrc/msm.cu: msm_count, the bin scan, msm_partition, msm_bin_sort and
msm_big_*), with the kernels' constants, plus the scratch-arena size of msm_run_batch before and after the two-level sort.

Layout: bucket b (0-based, digit magnitude - 1) of bucket set s has id s*B + b; its coarse bin is s*K + (b >> FB) with
FB = min(8, c - 1) fine bits and K = B >> FB bins per set.  Entries are (i + w*stride) | sign << 31."""
import numpy as np

R = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001

SORT_T = 512
PART_T = 512
PART_TILE = PART_T * 16        # digits per msm_partition block
SORT_FB_MAX = 8                # fine key = one byte
SORT_BIG = 1 << 17             # bins above this take the multi-block path
COUNT_LOCAL_MAX = 28672        # bins one msm_count block counts in shared memory
SCAN_TILE = 256 * 16
ACC_L_DEFAULT = 256
XYZZ_BYTES, SIGN = 128, 1 << 31


def recode_counts(s, c):
    """non-zero signed digits of one scalar (the entries it contributes)"""
    W, mask, half = 254 // c + 1, (1 << c) - 1, 1 << (c - 1)
    cnt, carry = 0, 0
    for _ in range(W):
        v = (s & mask) + carry
        s >>= c
        carry = 1 if v > half else 0
        cnt += ((1 << c) - v if v > half else v) != 0
    return cnt


def digits(vals, c):
    """signed digits of canonical scalars (Python ints) as the device encodes them: (W, n) uint32, magnitude | sign << 31"""
    n, W = len(vals), 254 // c + 1
    limbs = np.array([[(v >> (64 * k)) & (2**64 - 1) for k in range(4)] for v in vals], dtype=np.uint64).reshape(n, 4)
    limbs = np.concatenate([limbs, np.zeros((n, 1), np.uint64)], axis=1)
    mask, half = (1 << c) - 1, 1 << (c - 1)
    out = np.zeros((W, n), np.uint32)
    carry = np.zeros(n, np.uint64)
    for w in range(W):
        off = w * c
        q, r = divmod(off, 64)
        raw = limbs[:, q] >> np.uint64(r)
        if r + c > 64:
            raw |= limbs[:, q + 1] << np.uint64(64 - r)
        v = (raw & np.uint64(mask)) + carry
        neg = v > half
        mag = np.where(neg, np.uint64(1 << c) - v, v).astype(np.uint32)
        out[w] = mag | np.where(neg & (mag != 0), np.uint32(SIGN), np.uint32(0))
        carry = neg.astype(np.uint64)
    return out


class Plan:
    def __init__(self, n, c, batch=1, precomputed=False, stride=0):
        self.n, self.c, self.batch = n, c, batch
        self.W, self.B = 254 // c + 1, 1 << (c - 1)
        self.Ws = 1 if precomputed else self.W
        self.stride = stride if precomputed else 0
        self.NB = batch * self.Ws * self.B
        self.max_entries = n * self.W * batch
        self.FB = min(c - 1, SORT_FB_MAX)
        self.F = 1 << self.FB
        self.K = self.B >> self.FB
        self.wpg = self.W if self.Ws == 1 else max(1, min(COUNT_LOCAL_MAX // self.K, self.W))
        self.groups = -(-self.W // self.wpg)
        self.nbins = self.NB >> self.FB
        self.max_big = self.max_entries // SORT_BIG + 1


def entry_keys(pl, cols_digits):
    """(bucket id, entry) of every non-zero digit, in (column, window, index) order"""
    keys, ents = [], []
    for col, dg in enumerate(cols_digits):
        for w in range(pl.W):
            d = dg[w]
            i = np.nonzero(d)[0]
            mag = (d[i] & 0x7FFFFFFF).astype(np.int64) - 1
            s = col * pl.Ws + (0 if pl.Ws == 1 else w)
            keys.append(s * pl.B + mag)
            ents.append(((i + w * pl.stride).astype(np.uint64) | (d[i] & SIGN).astype(np.uint64)).astype(np.uint32))
    return np.concatenate(keys), np.concatenate(ents)


def plain_counting_sort(pl, cols_digits):
    keys, ents = entry_keys(pl, cols_digits)
    hist = np.bincount(keys, minlength=pl.NB)
    offsets = np.zeros(pl.NB + 1, np.int64)
    offsets[1:] = np.cumsum(hist)
    order = np.argsort(keys, kind="stable")
    return offsets, ents[order]


def two_level_sort(pl, cols_digits, big_blocks=264):
    """the kernels' schedule: bin counts (msm_count), bin scan, tile-by-tile runs (msm_partition, blocks taken in launch
    order), then each bin counting-sorted by its fine key, in one block or (above SORT_BIG) split over big_blocks slices"""
    bin_cnt = np.zeros(pl.nbins, np.int64)
    for col, dg in enumerate(cols_digits):
        for g in range(pl.groups):
            for w in range(g * pl.wpg, min(pl.W, (g + 1) * pl.wpg)):
                d = dg[w][dg[w] != 0]
                s = col * pl.Ws + (0 if pl.Ws == 1 else w)
                bins = ((d & 0x7FFFFFFF).astype(np.int64) - 1) >> pl.FB
                np.add.at(bin_cnt, s * pl.K + bins, 1)
    bin_off = np.zeros(pl.nbins + 1, np.int64)
    bin_off[1:] = np.cumsum(bin_cnt)
    M = int(bin_off[-1])
    cur = bin_off[:-1].copy()
    staged = np.zeros(M, np.uint32)
    fine = np.zeros(M, np.uint8)
    for col, dg in enumerate(cols_digits):
        for w in range(pl.W):
            s = col * pl.Ws + (0 if pl.Ws == 1 else w)
            for t0 in range(0, pl.n, PART_TILE):
                d = dg[w][t0:t0 + PART_TILE]
                i = np.nonzero(d)[0]
                bk = (d[i] & 0x7FFFFFFF).astype(np.int64) - 1
                sb = s * pl.K + (bk >> pl.FB)
                for b in np.unique(sb):  # one reservation per (tile, bin), entries in any order inside it
                    sel = sb == b
                    k = int(sel.sum())
                    pos = np.arange(cur[b], cur[b] + k)
                    cur[b] += k
                    gi = i[sel] + t0
                    staged[pos] = ((gi + w * pl.stride).astype(np.uint64) | (d[i[sel]] & SIGN)).astype(np.uint32)
                    fine[pos] = (bk[sel] & (pl.F - 1)).astype(np.uint8)
    assert np.array_equal(cur, bin_off[1:]), "every bin filled exactly"
    offsets = np.zeros(pl.NB + 1, np.int64)
    offsets[pl.NB] = M
    entries = np.zeros(M, np.uint32)
    big = []
    for sb in range(pl.nbins):
        lo, hi = int(bin_off[sb]), int(bin_off[sb + 1])
        if hi - lo > SORT_BIG:
            big.append(sb)
            continue
        f = fine[lo:hi]
        cnt = np.bincount(f, minlength=pl.F)
        base = lo + np.concatenate([[0], np.cumsum(cnt)[:-1]])
        offsets[sb * pl.F:(sb + 1) * pl.F] = base
        order = np.argsort(f, kind="stable")
        entries[lo:hi] = staged[lo:hi][order]
    for sb in big:  # msm_big_count totals, then per slice one reservation per bucket on the cursor
        lo, hi = int(bin_off[sb]), int(bin_off[sb + 1])
        tot = np.bincount(fine[lo:hi], minlength=pl.F)
        base = lo + np.concatenate([[0], np.cumsum(tot)[:-1]])
        offsets[sb * pl.F:(sb + 1) * pl.F] = base
        taken = np.zeros(pl.F, np.int64)
        for b in range(big_blocks):
            a = lo + (hi - lo) * b // big_blocks
            e = lo + (hi - lo) * (b + 1) // big_blocks
            f = fine[a:e]
            for v in np.unique(f):
                sel = f == v
                k = int(sel.sum())
                entries[base[v] + taken[v]:base[v] + taken[v] + k] = staged[a:e][sel]
                taken[v] += k
        assert np.array_equal(taken, tot)
    return offsets, entries, big


def _align(v, a=256):
    return (v + a - 1) // a * a


def _common_tail(pl, acc_l):
    nthreads = max(1, -(-pl.max_entries // acc_l))
    nthreads2 = -(-2 * nthreads // 64)
    kc = pl.c // 2
    rows, cols = pl.B >> kc, 1 << kc
    q_max = 0
    while (1 << q_max) < max(rows, cols):
        q_max += 1
    sets = pl.batch * pl.Ws
    return nthreads, nthreads2, sets * (rows + cols), 2 * (q_max + 1) * sets


def arena_bytes_parent(pl, acc_l=ACC_L_DEFAULT):
    """msm_run_batch's carve with the global-atomic sort (hist, offsets, cursor; digits + entries)"""
    nthreads, nthreads2, red_len, sums = _common_tail(pl, acc_l)
    ntiles = -(-pl.NB // SCAN_TILE)
    parts = [4 * (pl.NB + 1)] * 3 + [4 * (ntiles + 1), 256, 4 * (pl.max_entries + 4), 4 * (pl.max_entries + 4),
                                     XYZZ_BYTES * pl.NB, 4 * 2 * nthreads, XYZZ_BYTES * 2 * nthreads, 4 * 2 * nthreads2,
                                     XYZZ_BYTES * 2 * nthreads2, XYZZ_BYTES * red_len, XYZZ_BYTES * sums]
    return sum(_align(p) for p in parts)


def arena_bytes(pl, acc_l=ACC_L_DEFAULT):
    """msm_run_batch's carve with the two-level sort: the fine keys share the accumulate's partial records"""
    nthreads, nthreads2, red_len, sums = _common_tail(pl, acc_l)
    ntiles = -(-pl.nbins // SCAN_TILE)
    pval = max(XYZZ_BYTES * 2 * nthreads, pl.max_entries + 16)
    parts = [4 * (pl.NB + 1)] + [4 * (pl.nbins + 1)] * 3 + [4 * (pl.max_big + 1), 4 * 2 * pl.F * pl.max_big,
                                                            4 * (ntiles + 1), 256, 4 * (pl.max_entries + 4),
                                                            4 * (pl.max_entries + 4), XYZZ_BYTES * pl.NB, 4 * 2 * nthreads,
                                                            pval, 4 * 2 * nthreads2, XYZZ_BYTES * 2 * nthreads2,
                                                            XYZZ_BYTES * red_len, XYZZ_BYTES * sums]
    return sum(_align(p) for p in parts)


def max_batch(n, c):
    """msm_max_batch: columns one pipeline takes"""
    per_col = max(n, 1) * (254 // c + 1)
    return max(1, min(32, (1 << 28) // per_col))

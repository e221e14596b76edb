"""The two-level bucket sort of the device MSM (csrc/msm.cu), run as a numpy model with the kernels' bin split, tile size and
big-bin rule, must give exactly the offsets of a plain counting sort and, bucket by bucket, the same entries; its scratch
arena must not exceed the one of the global-atomic sort it replaced for the plans the bench runs."""
import random

import numpy as np
import pytest

import msm_sort_model as S


def columns(kind, n, seed):
    rng = random.Random(seed)
    if kind == "zero":
        return [0] * n
    if kind == "single":
        v = rng.randrange(S.R)
        return [v] * n
    if kind == "witness":  # ~60 % zero, ~30 % below 2^16, the rest uniform
        out = []
        for _ in range(n):
            u = rng.random()
            out.append(0 if u < 0.6 else (rng.randrange(1 << 16) if u < 0.9 else rng.randrange(S.R)))
        return out
    return [rng.randrange(S.R) for _ in range(n)]


def check(pl, vals_per_col, big_blocks=264):
    dg = [S.digits(v, pl.c) for v in vals_per_col]
    for v, d in zip(vals_per_col[:1], dg[:1]):  # the vectorised recoding counts what the scalar recoding counts
        assert int((d != 0).sum()) == sum(S.recode_counts(x, pl.c) for x in v)
    off_p, ent_p = S.plain_counting_sort(pl, dg)
    off_t, ent_t, big = S.two_level_sort(pl, dg, big_blocks)
    assert np.array_equal(off_p, off_t)
    for b in np.nonzero(np.diff(off_p))[0]:
        lo, hi = off_p[b], off_p[b + 1]
        assert np.array_equal(np.sort(ent_p[lo:hi]), np.sort(ent_t[lo:hi])), b
    return big


@pytest.mark.parametrize("kind", ["uniform", "witness", "single", "zero"])
@pytest.mark.parametrize("c", [2, 5, 9, 12])
def test_plain_bases_match_counting_sort(kind, c):
    n = S.PART_TILE + 37  # one full tile and a ragged one
    check(S.Plan(n, c), [columns(kind, n, 10 * c + len(kind))])


@pytest.mark.parametrize("c", [9, 13])
def test_precomputed_batch_matches_counting_sort(c):
    n = 3000
    kinds = ["uniform", "witness", "zero", "single", "witness"]
    pl = S.Plan(n, c, batch=len(kinds), precomputed=True, stride=n + 11)
    check(pl, [columns(k, n, 77 + j) for j, k in enumerate(kinds)])


def test_windows_beyond_one_count_group():
    """c = 21 plain: 13 windows of 4096 bins do not fit one block's counters, msm_count runs in window groups"""
    pl = S.Plan(700, 21)
    assert pl.groups == 2 and pl.wpg == 7
    check(pl, [columns("uniform", 700, 5)])
    pl = S.Plan(50, 24)
    assert pl.groups == pl.W and pl.K == 1 << 15
    check(pl, [columns("witness", 50, 6)])


def test_giant_bin_takes_the_multi_block_path():
    """one repeated scalar over more than SORT_BIG scalars: every window's bin is big; a batch beside ordinary columns"""
    n = S.SORT_BIG + 1000
    pl = S.Plan(n, 9, batch=2, precomputed=True, stride=n)
    big = check(pl, [[123456789] * n, columns("uniform", n, 9)], big_blocks=7)
    assert len(big) >= 1


@pytest.mark.parametrize("n,c,pre", [(1 << 20, 17, True), (1 << 24, 19, False), (1 << 25, 20, False)])
def test_arena_does_not_grow_for_the_bench_plans(n, c, pre):
    """at most 8 B per entry slot (digits + entries) plus O(NB) and O(blocks x bins): the fine keys share the partial
    records, hist and cursor are gone; the new arena is no larger than the old one"""
    batch = S.max_batch(n, c) if pre else 1
    pl = S.Plan(n, c, batch=batch, precomputed=pre, stride=n)
    new, old = S.arena_bytes(pl), S.arena_bytes_parent(pl)
    assert new <= old, (new, old)
    slots = pl.max_entries
    sort_extra = new - old + 8 * slots  # everything the sort needs beyond the accumulate's own arrays
    assert sort_extra <= 8 * slots + 64 * pl.NB

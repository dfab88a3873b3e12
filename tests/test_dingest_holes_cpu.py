"""The hole-mode key rule of the K5 group-by (csrc/group_kernels.cu), restated on numpy: a hole (agg == ~0, a record the device
decode dropped) gets the key n_agg, the radix bits cover n_agg itself, the LSD passes are stable. Then the holes sort behind
every live record, fall outside every CSR segment, are not counted as bad records, and the fold of the CSR is the fold of the
poll without its holes.

This file checks a model of the rule, not the kernel: the kernel is held to it on the GPU by tests/test_gpu_dingest_programs.py,
whose tables have power-of-two sizes, where a hole key with too few radix bits would fall among aggregate 0's records."""
import numpy as np
import pytest

from oracle import program_interp as I

HOLE = np.uint64(0xFFFFFFFFFFFFFFFF)


def group_with_holes(agg, n_agg):
    """(order, offsets, n_holes, n_bad) as K5 computes them in hole mode: LSD radix passes of 8 bits over the u32 keys."""
    hole = agg == HOLE
    bad = int(((agg >= n_agg) & ~hole).sum())
    keys = np.where(hole, np.uint64(n_agg), agg).astype(np.uint32)
    bits = 1
    while bits < 32 and (1 << bits) < n_agg + 1:
        bits += 1
    order = np.arange(len(keys))
    for shift in range(0, bits, 8):
        digit = (keys[order] >> np.uint32(shift)) & np.uint32(255)
        order = order[np.argsort(digit, kind="stable")]
    n_live = len(keys) - int(hole.sum())
    sorted_keys = keys[order]
    offsets = np.searchsorted(sorted_keys[:n_live], np.arange(n_agg + 1), side="left") * 64
    return order, offsets, int(hole.sum()), bad, sorted_keys


@pytest.mark.parametrize("n_agg", [1, 255, 256, 257, 65536, 70000])
def test_holes_sort_last_and_stay_out_of_the_csr(n_agg):
    rng = np.random.default_rng(n_agg)
    n = 5000
    agg = rng.integers(0, n_agg, size=n).astype(np.uint64)
    agg[rng.random(n) < 0.1] = HOLE
    order, offsets, n_holes, bad, sorted_keys = group_with_holes(agg, n_agg)
    n_live = n - n_holes
    assert bad == 0
    assert (agg[order[n_live:]] == HOLE).all() and (agg[order[:n_live]] != HOLE).all()
    assert (np.diff(sorted_keys.astype(np.int64)) >= 0).all()
    assert offsets[-1] == 64 * n_live                      # the CSR ends before the first hole
    for a in np.unique(agg[agg != HOLE])[:50]:
        seg = order[offsets[a] // 64:offsets[a + 1] // 64]
        assert (agg[seg] == a).all() and (np.diff(seg) > 0).all()   # the aggregate's records, in arrival order


def test_bits_must_cover_the_hole_key():
    """With n_agg = 256 eight bits hold every live key but not the hole key 256: sorted on those bits alone, holes would land
    among the records of aggregate 0."""
    agg = np.array([0, 0xFFFFFFFFFFFFFFFF, 0, 1], dtype=np.uint64)
    keys = np.where(agg == HOLE, np.uint64(256), agg).astype(np.uint32)
    order8 = np.argsort(keys & np.uint32(255), kind="stable")
    assert (agg[order8[:3]] == np.array([0, HOLE, 0], dtype=np.uint64)).all()
    order, _, _, _, _ = group_with_holes(agg, 256)
    assert agg[order[-1]] == HOLE


def test_out_of_range_records_are_bad_and_holes_are_not():
    agg = np.array([3, 0xFFFFFFFFFFFFFFFF, 7, 10, 0xFFFFFFFFFFFFFFFF], dtype=np.uint64)
    _, _, n_holes, bad, _ = group_with_holes(agg, 8)
    assert (n_holes, bad) == (2, 1)


def test_fold_of_the_csr_is_the_fold_without_holes():
    rules = [(I.CREATE, [(I.OP_SET, 0, 16, 8)]), (I.IF_EXISTS, [(I.OP_ADD_I32, 8, 20, 4)]), (I.THROW, [])]
    rng = np.random.default_rng(5)
    n, n_agg = 400, 37
    rec = rng.integers(0, 256, size=(n, 64), dtype=np.uint8)
    rec[:, 0:4] = rng.choice([0, 1, 1, 1, 2], size=n).astype(np.uint32).view(np.uint8).reshape(-1, 4)
    agg = rng.integers(0, n_agg, size=n).astype(np.uint64)
    agg[rng.random(n) < 0.2] = HOLE
    rec[:, 8:16] = agg.view(np.uint8).reshape(-1, 8)
    states = np.zeros((n_agg, 24), np.uint8)
    order, offsets, n_holes, _, _ = group_with_holes(agg, n_agg)
    grouped = rec[order[:n - n_holes]]
    got = I.fold(rules, 24, grouped, offsets, states)
    want = I.fold_arrival_order(rules, 24, rec[agg != HOLE], states)
    assert np.array_equal(got, want)

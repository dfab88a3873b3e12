"""-m gpu: fold programs at the sizes where the kernels' structure actually runs, against the compiled program oracle.

tests/test_gpu_program_fuzz.py folds a few thousand records per program: there fold_runs.cu launches a handful of warps
and each folds one step. Here every W = 2 fixed-record log holds 8.4 M records (538 MB). An H100 keeps at most
132 SMs x 64 warps = 8 448 warps resident, the runs kernel's grid is capped at what is co-resident, and one step is
32 * R records with R <= 8, so the log is at least 8.4e6 / (32 * 8) = 32 812 steps: every warp folds at least 3 steps even
at R = 8, and look-back chains cross many spans without a segment head. The logs also carry runs of 3 000 empty segments
at the start, middle and end, segments aligned on step and span multiples, one segment of exactly one step, a hot
aggregate with a quarter of the log (a throw as its first record), a second one with a throw as its last record, a
64-step segment without a throw (so no replay hides a wrong look-back), MatchError types from n_types up to 2^32 - 1, and a CSR that starts at a non-zero offset.

Programs are built so the kernel instantiation is known by construction (oracle/program_corpus.py row_program: a fixed
number of distinct source words, hence n_slots). Every case compares the whole state table byte for byte with
oracle/program_oracle.c, and stats().n_events / n_errors where the engine reports them. Each log is loaded once; kernels
and options vary through set_option and set_initial_states(None).
"""
import numpy as np
import pytest

from oracle import program_corpus as PC
from oracle import program_interp as I
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P

pytestmark = pytest.mark.gpu

N_REC = 8_400_000          # per W = 2 log: >= 3 steps per resident warp at R = 8 (see the module docstring)
N_AGG = 1_000_000
PAD = 7                    # records in front of the first segment
N_RUN_VARIANTS = 7
NAN = float("nan")


def same(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(want)} states differ; first {bad[:6]}\n got {got[bad[0]].tolist()}\nwant {want[bad[0]].tolist()}")


def check(e, want, nev, nerr, what):
    same(e.export_states(), want, what)
    st = e.stats()
    assert (st.n_events, st.n_errors) == (nev, nerr), f"{what}: stats (n_events, n_errors) = {(st.n_events, st.n_errors)}, oracle {(nev, nerr)}"


def throw_type(rules):
    return next((t for t, (ex, _) in enumerate(rules) if ex == I.THROW), len(rules))


def shaped_fixed_log(seed, rules, n_rec=N_REC, n_agg=N_AGG, f64_offsets=(), f64_values=PC.SPECIAL_F64):
    rng = np.random.default_rng(seed)
    counts, hot, hot2 = PC.shaped_counts(rng, n_agg, n_rec)
    buf, seg, _ = PC.fixed_log(rng, rules, counts, f64_offsets=f64_offsets, f64_values=f64_values, pad_records=PAD)
    PC.set_type(buf, seg, hot, 0, throw_type(rules))            # throws as the first record of the hot aggregate
    PC.set_type(buf, seg, hot2, -1, len(rules))                 # ... and as the last record of the second one
    # the next longest segment (64 steps of 256 records, several spans) gets no throw: its state is not replayed, only the
    # look-back carries it across the spans that hold no segment head
    lens = np.diff(seg.astype(np.int64)) // 64
    lens[[hot, hot2]] = 0
    calm = int(np.argmax(lens))
    rows = buf[int(seg[calm]) // 64:int(seg[calm + 1]) // 64]
    types = rows[:, 0:4].copy().view(np.uint32).ravel()
    rows[np.isin(types, [t for t, (ex, _) in enumerate(rules) if ex == I.THROW]) | (types >= len(rules)), 0:4] = 0
    return buf, seg


def oracle_fixed(rules, sb, buf, seg, prior=None, f64=()):
    return I.c_fold(rules, sb, buf.reshape(-1)[int(seg[0]):], seg, initial=prior, f64_fields=f64)


def fold_fixed(e, kernel, prior=None, **options):
    e.set_option("kernel", kernel)
    for k, v in options.items():
        e.set_option(k, v)
    e.set_initial_states(prior)
    e.fold()


# ------------------------------------------------------------------ record-parallel families (transformer algebra)
FAMILIES = [  # name, state words W, class, distinct source words, every run variant
    ("w2_class0_ns2", 2, 0, 1, True),
    ("w2_class0_ns3", 2, 0, 2, True),
    ("w2_class0_ns6", 2, 0, 5, True),
    ("w2_class0_direct_ns9", 2, 0, 8, False),
    ("w2_class1", 2, 1, 3, False),
    ("w6_class0", 6, 0, 6, False),
    ("w6_class1", 6, 1, 6, False),
]


@pytest.mark.parametrize("name,W,cls,n_src,variants", FAMILIES, ids=[f[0] for f in FAMILIES])
def test_row_program_family_at_scale(name, W, cls, n_src, variants):
    seed = 52000 + sum(map(ord, name))
    rng = np.random.default_rng(seed)
    rules = PC.row_program(rng, W, cls, n_src)
    sb = 4 * W + 8
    buf, seg = shaped_fixed_log(seed + 1, rules)
    want, nev, nerr = oracle_fixed(rules, sb, buf, seg)
    assert nerr > 500 and nev > N_REC // 2
    what = f"{name} rules {rules}"
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_FIXED64, rules))
        e.load_events(buf, seg)
        for v in range(N_RUN_VARIANTS) if variants else [0]:
            fold_fixed(e, 2, run_variant=v)          # forced runs kernel: must accept every program of the family
            check(e, want, nev, nerr, f"{what} runs kernel variant {v}")
        e.set_option("run_variant", 0)
        kernels = [0, 1] + ([3] if W == 2 and cls == 0 and n_src <= 5 else [])
        for kernel in kernels:
            fold_fixed(e, kernel)
            check(e, want, nev, nerr, f"{what} kernel {kernel}")
        # the same log on top of its own output (prior states, publish rule against them)
        want2, nev2, nerr2 = oracle_fixed(rules, sb, buf, seg, prior=want)
        for kernel in [2, 1] + ([3] if 3 in kernels else []):
            fold_fixed(e, kernel, prior=want)
            check(e, want2, nev2, nerr2, f"{what} kernel {kernel} with prior states")


def w14_double_program():
    """64-byte states, class 1, a JVM Double at +8 (record +24): CREATE builds, IF_EXISTS copies the Double alone, adds,
    or hands the instance back."""
    rules = [
        (I.CREATE, [(I.OP_SET, 0, 16, 8), (I.OP_SET, 8, 24, 8), (I.OP_SET, 16, 32, 16), (I.OP_ADD_I32, 40, 4, 4)]),
        (I.IF_EXISTS, [(I.OP_SET, 8, 24, 8)]),
        (I.IF_EXISTS, []),
        (I.IF_EXISTS, [(I.OP_ADD_I32, 16, 48, 4), (I.OP_SUB_I32, 44, 52, 4), (I.OP_SET, 48, 56, 8)]),
        (I.TOMBSTONE, []),
        (I.THROW, []),
    ]
    return rules, [8]


def test_w14_class1_double_field_at_scale():
    """NaN, -0.0 and the instance rule: a segment that only copies the same NaN bits over a NaN state builds a new
    instance (published: NaN != NaN); one that only hands the instance back is not published."""
    rules, f64 = w14_double_program()
    sb = 64
    vals = [NAN, 0.0, -0.0, 1.5]
    buf, seg = shaped_fixed_log(53001, rules, n_rec=4_200_000, n_agg=700_000, f64_offsets=[24], f64_values=vals)
    want, nev, nerr = oracle_fixed(rules, sb, buf, seg, f64=f64)
    # a prior table that mixes None, existing and NaN rows
    prior = want.copy()
    rng = np.random.default_rng(53002)
    rows = rng.random(len(prior))
    prior[rows < 0.2] = 0
    nan_rows = (rows >= 0.2) & (rows < 0.5)
    prior[nan_rows, 8:16] = np.frombuffer(np.float64(NAN).tobytes(), np.uint8)
    prior[nan_rows, 56] = I.ST_EXISTS
    prior[:, 57:] = 0
    want2, nev2, nerr2 = oracle_fixed(rules, sb, buf, seg, prior=prior, f64=f64)
    changed = want2[:, 56] & I.ST_CHANGED
    assert (changed[nan_rows] == 0).any() and (changed[nan_rows] != 0).any()
    what = f"W14 class 1 f64 rules {rules}"
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_FIXED64, rules, f64_fields=f64))
        e.load_events(buf, seg)
        for kernel in (2, 0, 1):
            fold_fixed(e, kernel)
            check(e, want, nev, nerr, f"{what} kernel {kernel}")
            fold_fixed(e, kernel, prior=prior)
            check(e, want2, nev2, nerr2, f"{what} kernel {kernel} on a mixed prior table")
        # a fold on top of its own output
        want3, nev3, nerr3 = oracle_fixed(rules, sb, buf, seg, prior=want2, f64=f64)
        fold_fixed(e, 2, prior=e.export_states())
        check(e, want3, nev3, nerr3, f"{what} folded twice")


# ------------------------------------------------------------------ outside the algebra: the lane-sequential kernel
OUTSIDE = {
    "i64_adds_16B": (16, [(I.MATERIALISE, [(I.OP_ADD_I64, 0, 16, 8)]), (I.MATERIALISE, [(I.OP_SUB_I64, 0, 24, 8)]),
                          (I.CREATE, [(I.OP_SET, 0, 4, 4)]), (I.THROW, [])]),
    "materialise_and_if_exists_32B": (32, [(I.CREATE, [(I.OP_SET, 0, 16, 8)]), (I.MATERIALISE, [(I.OP_ADD_I32, 8, 20, 4)]),
                                           (I.IF_EXISTS, [(I.OP_SET, 12, 4, 4)]), (I.TOMBSTONE, []), (I.THROW, [])]),
    "state_48B": (48, [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4), (I.OP_SET, 24, 32, 16)]),
                       (I.CREATE, [(I.OP_SET, 8, 20, 16)]), (I.TOMBSTONE, []), (I.THROW, [])]),
    "state_128B": (128, [(I.CREATE, [(I.OP_SET, 0, 16, 48), (I.OP_SET, 64, 16, 48)]), (I.IF_EXISTS, [(I.OP_ADD_I64, 112, 24, 8)]),
                         (I.IF_EXISTS, []), (I.THROW, [])]),
}


@pytest.mark.parametrize("name", list(OUTSIDE))
def test_program_outside_the_algebra_at_scale(name):
    sb, rules = OUTSIDE[name]
    buf, seg = shaped_fixed_log(54000 + sum(map(ord, name)), rules, n_rec=4_200_000, n_agg=500_000)
    want, nev, nerr = oracle_fixed(rules, sb, buf, seg)
    want2, nev2, nerr2 = oracle_fixed(rules, sb, buf, seg, prior=want)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_FIXED64, rules))
        e.load_events(buf, seg)
        for kernel in (2, 3):
            with pytest.raises(SgrError) as ei:
                fold_fixed(e, kernel)
            assert ei.value.code == N.SGR_ERR_UNSUPPORTED
        for variant in (range(6) if sb == 16 else [-1]):
            e.set_option("fold_variant", variant)
            for kernel in (0, 1):
                fold_fixed(e, kernel)
                check(e, want, nev, nerr, f"{name} kernel {kernel} fold_variant {variant}")
            fold_fixed(e, 0, prior=want)
            check(e, want2, nev2, nerr2, f"{name} fold_variant {variant} with prior states")
        e.set_option("fold_variant", -1)


# ------------------------------------------------------------------ arrival order
BULK = {
    "entry16": [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4)]), (I.MATERIALISE, [(I.OP_SUB_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4)]),
                (I.MATERIALISE, []), (I.THROW, [])],
    "entry32_tombstones": [(I.MATERIALISE, [(I.OP_SET, 0, 16, 4), (I.OP_SET, 4, 4, 4)]), (I.CREATE, [(I.OP_SET, 0, 20, 4)]),
                           (I.TOMBSTONE, []), (I.MATERIALISE, []), (I.THROW, [])],
    "add_only": [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 16, 4), (I.OP_SUB_I32, 4, 20, 4)]), (I.MATERIALISE, []), (I.THROW, [])],
}
# a word that one rule SETs and another ADDs: not a bulk layout, the three-phase micro-batch kernel
SET_AND_ADD = [(I.MATERIALISE, [(I.OP_SET, 0, 16, 4), (I.OP_ADD_I32, 4, 20, 4)]), (I.MATERIALISE, [(I.OP_ADD_I32, 0, 24, 4)]),
               (I.MATERIALISE, []), (I.THROW, [])]
N_SLOTS = 4_200_000        # 16-byte states + scratch: larger than the H100's 50 MB L2


def arrival_log(seed, rules, n_rec, n_agg, hot=5, hot_share=0.25):
    """Records in arrival order: aggregates drawn uniformly (a quarter of them for one hot aggregate), seq = position."""
    rng = np.random.default_rng(seed)
    aggs = rng.integers(0, n_agg, size=n_rec).astype(np.uint64)
    aggs[rng.random(n_rec) < hot_share] = hot
    rec = rng.integers(0, 256, size=(n_rec, 64), dtype=np.uint8)
    rec[:, 0:4] = PC.type_mix(rules, n_rec, rng, p_throw=1e-4).view(np.uint8).reshape(-1, 4)
    rec[:, 4:8] = np.arange(1, n_rec + 1, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
    rec[:, 8:16] = aggs.view(np.uint8).reshape(-1, 8)
    return rec


@pytest.mark.parametrize("layout", list(BULK))
def test_fold_unsorted_bulk_layouts(layout):
    rules = BULK[layout]
    big = arrival_log(55001, rules, 8_400_000, N_SLOTS)
    small = arrival_log(55002, rules, 1_000_000, N_SLOTS)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        for which, rec in (("log larger than the table", big), ("log smaller than the table", small)):
            want, nev, nerr = I.c_fold_arrival_order(rules, 16, rec, None, n_agg=N_SLOTS)
            assert nerr > 0
            for bulk in (1, 0):
                e.set_option("bulk", bulk)
                e.fold_unsorted(rec, N_SLOTS)
                check(e, want, nev, nerr, f"{layout} {which} bulk={bulk}")
        e.set_option("bulk", 1)
        want, nev, nerr = I.c_fold_arrival_order(rules, 16, big, None, n_agg=N_SLOTS)
        try:
            for bps in (1, 8, 32):
                e.set_option("bulk_blocks_per_sm", bps)
                e.fold_unsorted(big, N_SLOTS)
                check(e, want, nev, nerr, f"{layout} bulk_blocks_per_sm={bps}")
        finally:
            e.set_option("bulk_blocks_per_sm", 0)
        # a bulk fold refused for an out-of-range aggregate leaves the scratch clean for the next one
        bad = small.copy()
        bad[len(bad) // 2, 8:16] = np.frombuffer(np.uint64(N_SLOTS).tobytes(), np.uint8)
        with pytest.raises(SgrError) as ei:
            e.fold_unsorted(bad, N_SLOTS)
        assert ei.value.code == N.SGR_ERR_INVALID
        want_s, nev_s, nerr_s = I.c_fold_arrival_order(rules, 16, small, None, n_agg=N_SLOTS)
        e.fold_unsorted(small, N_SLOTS)
        check(e, want_s, nev_s, nerr_s, f"{layout} after a refused bulk fold")


def test_set_and_added_word_and_micro_batches():
    """The three-phase micro-batch kernel from None, then micro-batches larger and smaller than the table (finishing by
    slot and by record), against the oracle after every batch."""
    rules = SET_AND_ADD
    n_agg = 1_000_000
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        first = arrival_log(56001, rules, 4_000_000, n_agg)
        table, nev, nerr = I.c_fold_arrival_order(rules, 16, first, None, n_agg=n_agg)
        e.fold_unsorted(first, n_agg)
        check(e, table, nev, nerr, "three-phase fold_unsorted")
        for b, n in enumerate([3_000_000, 20_000, 1_500_000, 300]):
            batch = arrival_log(56010 + b, rules, n, n_agg, hot=int(7 + b))
            table, nev, nerr = I.c_fold_arrival_order(rules, 16, batch, table)
            e.fold_incremental(batch)
            check(e, table, nev, nerr, f"three-phase micro-batch {b} ({n} records)")


@pytest.mark.parametrize("n_agg", [256, 257, (1 << 24) + 3])
def test_group_by_radix_passes(n_agg):
    """A program outside the sort-free class through the stable group-by: one, two and four radix passes."""
    sb, rules = OUTSIDE["materialise_and_if_exists_32B"]
    n_rec = 3_000_000
    rec = arrival_log(57000 + n_agg % 1000, rules, n_rec, n_agg, hot=n_agg - 1, hot_share=0.05)
    k = min(1000, n_agg)                                           # the highest aggregate indices all occur
    rec[-k:, 8:16] = np.arange(n_agg - k, n_agg, dtype=np.uint64).view(np.uint8).reshape(-1, 8)
    want, nev, nerr = I.c_fold_arrival_order(rules, sb, rec, None, n_agg=n_agg)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_FIXED64, rules))
        e.fold_unsorted(rec, n_agg)
        check(e, want, nev, nerr, f"group-by n_agg={n_agg}")


# ------------------------------------------------------------------ variable records
@pytest.mark.parametrize("max_record_bytes,n_rec", [(528, 2_000_000), (1040, 600_000), (2064, 300_000)])
def test_variable_records_at_scale(max_record_bytes, n_rec):
    rng = np.random.default_rng(58000 + max_record_bytes)
    rules = PC.row_program(rng, 2, 0, 3)                           # 16-byte class 0: the record-parallel vruns kernel
    counts, _, _ = PC.shaped_counts(rng, n_rec // 8, n_rec, empty_run=500)
    buf, seg, rec_off = PC.var_log(rng, rules, counts, max_record_bytes - 16)
    want, nev, nerr = I.c_fold_var(rules, 16, buf, seg, max_record_bytes=max_record_bytes)
    assert nerr > 0
    what = f"var cap {max_record_bytes} rules {rules}"
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_VAR16, rules))
        e.set_option("max_record_bytes", max_record_bytes)
        e.load_events_indexed(buf, seg, rec_off)
        for stages in (1, 2, 3):
            e.set_option("var_stages", stages)
            for stage_bytes in (12288, 4096):               # 4096 < 32 x the largest record
                e.set_option("var_stage_bytes", stage_bytes)
                fold_fixed(e, 0)
                check(e, want, nev, nerr, f"{what} with directory, var_stages {stages}, var_stage_bytes {stage_bytes}")
        e.set_option("var_stages", 1); e.set_option("var_stage_bytes", 12288)
        e.load_events(buf, seg)                             # no directory: the lane-sequential kernel
        for kernel in (0, 1):
            fold_fixed(e, kernel)
            check(e, want, nev, nerr, f"{what} without directory, kernel {kernel}")
    # a program outside the record-parallel class on the same log
    sb, rules2 = 32, [(I.CREATE, [(I.OP_SET, 0, 16, 8), (I.OP_ADD_I32, 8, 60, 4)]), (I.IF_EXISTS, [(I.OP_SET, 12, 72, 12)]),
                      (I.TOMBSTONE, []), (I.THROW, [])]
    want2, nev2, nerr2 = I.c_fold_var(rules2, sb, buf, seg, max_record_bytes=max_record_bytes)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_VAR16, rules2))
        e.set_option("max_record_bytes", max_record_bytes)
        e.load_events(buf, seg)
        fold_fixed(e, 0)
        check(e, want2, nev2, nerr2, f"var cap {max_record_bytes} rules {rules2}")


# ------------------------------------------------------------------ replay-list overflow
REDO_CAP = 1 << 20
OVERFLOW_RULES = [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4)]), (I.MATERIALISE, [(I.OP_SUB_I32, 0, 16, 4)]),
                  (I.THROW, [])]


def overflow_counts_and_types(rng, n_agg=1_200_000, per=3):
    """per records per aggregate; more than 2^20 aggregates throw at a record that is not their last."""
    types = rng.integers(0, 2, size=(n_agg, per)).astype(np.uint32)
    throwing = rng.permutation(n_agg)[:REDO_CAP + 60_000]
    types[throwing, rng.integers(0, per - 1, size=len(throwing))] = 2
    return np.full(n_agg, per, dtype=np.int64), types.ravel()


def test_replay_list_overflow_fixed_records():
    rng = np.random.default_rng(59001)
    counts, types = overflow_counts_and_types(rng)
    buf, seg, _ = PC.fixed_log(rng, OVERFLOW_RULES, counts, p_throw=0.0)
    buf[:, 0:4] = types.view(np.uint8).reshape(-1, 4)
    want, nev, nerr = I.c_fold(OVERFLOW_RULES, 16, buf, seg)
    assert nerr > REDO_CAP and nev < int(counts.sum())
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, OVERFLOW_RULES))
        e.load_events(buf, seg)
        for kernel in (0, 3):
            fold_fixed(e, kernel)
            check(e, want, nev, nerr, f"replay-list overflow, kernel {kernel}")
        # in place on prior states the kernel has already overwritten part of the table: refused, and the table is unreadable
        for kernel in (0, 3):
            e.set_option("kernel", kernel)
            e.set_initial_states(want)
            with pytest.raises(SgrError) as ei:
                e.fold()
            assert ei.value.code == N.SGR_ERR_UNSUPPORTED
            for read in (e.export_states, lambda: e.get("agg-0")):
                with pytest.raises(SgrError) as ei:
                    read()
                assert ei.value.code == N.SGR_ERR_STATE
            fold_fixed(e, kernel)
            check(e, want, nev, nerr, f"fresh fold after an overflow on prior states, kernel {kernel}")
        # the sort-based micro-batch path folds in place too
        e.set_option("kernel", 0)
        e.set_option("incremental", 1)
        batch = buf[PC.interleave(rng, np.repeat(np.arange(len(counts), dtype=np.uint64), counts))]
        with pytest.raises(SgrError) as ei:
            e.fold_incremental(batch)
        assert ei.value.code == N.SGR_ERR_UNSUPPORTED
        with pytest.raises(SgrError) as ei:
            e.export_states()
        assert ei.value.code == N.SGR_ERR_STATE
        e.set_option("incremental", 0)
        fold_fixed(e, 0)
        check(e, want, nev, nerr, "fresh fold after an overflow in a micro-batch")


def test_replay_list_overflow_variable_records():
    rng = np.random.default_rng(59002)
    counts, types = overflow_counts_and_types(rng)
    buf, seg, rec_off = PC.var_log(rng, OVERFLOW_RULES, counts, 96, p_short=0.0, p_throw=0.0, n_malformed=0)
    starts = rec_off[:-1].astype(np.int64)
    tb = types.view(np.uint8).reshape(-1, 4)
    for j in range(4):
        buf[starts + j] = tb[:, j]
    want, nev, nerr = I.c_fold_var(OVERFLOW_RULES, 16, buf, seg)
    assert nerr > REDO_CAP
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_VAR16, OVERFLOW_RULES))
        e.load_events_indexed(buf, seg, rec_off)
        fold_fixed(e, 0)
        check(e, want, nev, nerr, "replay-list overflow, vruns")

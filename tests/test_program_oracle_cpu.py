"""No GPU: the compiled fold-program oracle (oracle/program_oracle.c) equals the Python interpreter
(oracle/program_interp.py) and the sample-model oracle (oracle/sgr_oracle.c).

tests/test_gpu_program_scale.py checks the kernels against the compiled oracle at millions of records; this file is what
ties that oracle to the written semantics: the same random programs and logs through both restatements, byte for byte,
and its statistics against what the interpreter's table implies.
"""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import program_corpus as PC
from oracle import program_interp as I
from surge_b200 import programs as P
from surge_b200 import synth as S


def same(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(want)} states differ; first {bad[:6]}\n got {got[bad[0]].tolist()}\nwant {want[bad[0]].tolist()}")


def implied_stats(table, state_bytes, counts):
    """(n_events, n_errors) a fold table implies: a throwing aggregate applied err_idx events, any other all of them."""
    t = np.ascontiguousarray(table).reshape(-1, state_bytes)
    flags = t[:, state_bytes - 8:state_bytes - 4].copy().view(np.uint32).ravel()
    err = t[:, state_bytes - 4:].copy().view(np.uint32).ravel().astype(np.int64)
    threw = (flags & I.ST_ERROR) != 0
    return int(np.where(threw, err, np.asarray(counts, dtype=np.int64)).sum()), int(threw.sum())


def rules_of(prog):
    return [(int(prog.rules[t].exists_rule), [(int(o.opcode), int(o.dst_off), int(o.src_off), int(o.len))
                                               for o in list(prog.rules[t].ops)[:prog.rules[t].n_ops]]) for t in range(prog.n_types)]


@pytest.mark.parametrize("seed", range(160))
def test_fixed_records_match_the_interpreter(seed):
    """Random programs (every state width, 64-bit ops, f64 fields, all exists rules) on a CSR log, from None and on top
    of the first table, and a CSR that starts at a non-zero offset."""
    rng = np.random.default_rng(31000 + seed)
    state_bytes, rules, f64 = PC.draw_program(rng)
    rec, off, _ = PC.draw_log(rng, len(rules), 90, 150, f64)
    counts = np.diff(off.astype(np.int64)) // 64
    want = I.fold(rules, state_bytes, rec, off, f64_fields=f64)
    got, nev, nerr = I.c_fold(rules, state_bytes, rec, off, f64_fields=f64)
    what = f"seed {seed} state_bytes {state_bytes} rules {rules} f64 {f64}"
    same(got, want, what)
    assert (nev, nerr) == implied_stats(want, state_bytes, counts), what
    rec2, off2, _ = PC.draw_log(rng, len(rules), 90, 40, f64)
    off2 = off2 + 64 * 5                               # the records start at the first segment's offset
    want2 = I.fold(rules, state_bytes, rec2, off2, initial=want, f64_fields=f64)
    got2, nev2, nerr2 = I.c_fold(rules, state_bytes, rec2, off2, initial=want, f64_fields=f64)
    same(got2, want2, what + " with prior states")
    assert (nev2, nerr2) == implied_stats(want2, state_bytes, np.diff(off2.astype(np.int64)) // 64), what


def draw_granular_case(seed):
    """A random program on a CSR log at 16-byte granularity (oracle/program_corpus.py granular_log): the log starts at
    0, 16, 32 or 48 (mod 64), random segments end in a 16-, 32- or 48-byte partial record, and by seed the first, a middle
    and the last segment, the long segment and a segment of exactly 16 bytes do too. Returns (rng, state_bytes, rules,
    f64, log, seg_offsets, whole-record counts, tails)."""
    rng = np.random.default_rng(37000 + seed)
    state_bytes, rules, f64 = PC.draw_program(rng)
    rec, off, _ = PC.draw_log(rng, len(rules), 60, 100, f64)
    counts = np.diff(off.astype(np.int64)) // 64
    n_agg = len(counts)
    tails = np.where(rng.random(n_agg) < 0.2, 16 * rng.integers(1, 4, size=n_agg), 0)
    if seed % 7 == 6:
        tails[:] = 0                                       # whole records only, off the 64-byte grid by the start alone
    else:
        for i in ([0] if seed % 3 == 0 else []) + [n_agg // 2] + ([n_agg - 1] if seed % 3 == 1 else []):
            tails[i] = 16 * (1 + seed % 3)
        if seed % 4 == 1:
            tails[int(np.argmax(counts))] = 48            # a long segment that ends in a partial record
        if seed % 5 == 0:
            z = int(rng.integers(0, n_agg))
            rec = np.delete(rec, np.s_[int(counts[:z].sum()):int(counts[:z + 1].sum())], axis=0)
            counts[z], tails[z] = 0, 16                   # exactly 16 bytes: throws at err_idx 0
    start = 16 * (seed % 4) + 64 * int(rng.integers(0, 3))
    log, seg = PC.granular_log(rng, rec, counts, tails, start)
    return rng, state_bytes, rules, f64, log, seg, counts, tails


@pytest.mark.parametrize("seed", range(300))
def test_granular_fixed_logs_match_the_interpreter(seed):
    """Fixed records at 16-byte granularity (include/sgr.h): whole records fold at their byte positions, a trailing
    partial record throws at err_idx = the whole records before it, and the segments after it start off the 64-byte grid.
    The compiled oracle equals the interpreter from None and on top of the first table."""
    _, state_bytes, rules, f64, log, seg, counts, _ = draw_granular_case(seed)
    what = f"seed {seed} state_bytes {state_bytes} rules {rules} f64 {f64} start {int(seg[0])}"
    recs = log[int(seg[0]):]
    want = I.fold(rules, state_bytes, recs, seg, f64_fields=f64)
    got, nev, nerr = I.c_fold(rules, state_bytes, recs, seg, f64_fields=f64)
    same(got, want, what)
    assert (nev, nerr) == implied_stats(want, state_bytes, counts), what
    want2 = I.fold(rules, state_bytes, recs, seg, initial=want, f64_fields=f64)
    got2, nev2, nerr2 = I.c_fold(rules, state_bytes, recs, seg, initial=want, f64_fields=f64)
    same(got2, want2, what + " with prior states")
    assert (nev2, nerr2) == implied_stats(want2, state_bytes, counts), what


def test_granular_partial_records_throw_where_the_rule_says():
    """The rule itself, not only agreement between the two restatements: every segment that ends in a partial record is an
    error row at err_idx = its whole records unless an earlier record threw, its prior state kept; every 64-aligned log
    folds exactly as the same records packed from offset 0."""
    for seed in range(300):
        _, state_bytes, rules, f64, log, seg, counts, tails = draw_granular_case(seed)
        got, _, _ = I.c_fold(rules, state_bytes, log[int(seg[0]):], seg, f64_fields=f64)
        flags = got[:, state_bytes - 8:state_bytes - 4].copy().view(np.uint32).ravel()
        err = got[:, state_bytes - 4:].copy().view(np.uint32).ravel()
        part = tails > 0
        assert ((flags[part] & I.ST_ERROR) != 0).all(), f"seed {seed}"
        assert (err[part] <= counts[part]).all() and ((flags[part] & I.ST_EXISTS) == 0).all(), f"seed {seed}"
        if not part.any():
            starts = seg[:-1].astype(np.int64)
            packed = np.concatenate([log[s:s + 64 * c] for s, c in zip(starts, counts)] + [np.zeros(0, np.uint8)])
            off0 = np.zeros(len(counts) + 1, np.uint64)
            np.cumsum(64 * counts, out=off0[1:])
            want, _, _ = I.c_fold(rules, state_bytes, packed, off0, f64_fields=f64)
            same(got, want, f"seed {seed}: 16-byte start {int(seg[0])} against the packed log")


def test_the_granular_draws_cover_what_the_pin_claims():
    """Every log start mod 64, every tail length, partial records in the first, a middle and the last segment and at the
    end of the long one, a 16-byte segment, empty segments that start off the 64-byte grid, a partial record after a
    throw in the same segment, and logs of whole records at each unaligned start."""
    seen = set()
    for seed in range(300):
        _, state_bytes, rules, f64, log, seg, counts, tails = draw_granular_case(seed)
        rel = seg.astype(np.int64) - int(seg[0])
        seen.add(("start", int(seg[0]) % 64))
        seen.update(("tail", int(t)) for t in tails if t)
        if tails[0]:
            seen.add("first")
        if tails[-1]:
            seen.add("last")
        if tails[1:-1].any():
            seen.add("middle")
        if tails[int(np.argmax(counts))] and counts.max() >= 90:
            seen.add("long")
        if ((counts == 0) & (tails == 16)).any():
            seen.add("16 bytes")
        if ((np.diff(rel) == 0) & (rel[:-1] % 64 != 0)).any():
            seen.add("empty off grid")
        if not tails.any() and int(seg[0]) % 64:
            seen.add(("whole", int(seg[0]) % 64))
        got, _, _ = I.c_fold(rules, state_bytes, log[int(seg[0]):], seg, f64_fields=f64)
        err = got[:, state_bytes - 4:].copy().view(np.uint32).ravel()
        if ((tails > 0) & (err < counts)).any():
            seen.add("throw before a partial")
    assert {("start", s) for s in (0, 16, 32, 48)} <= seen
    assert {("tail", t) for t in (16, 32, 48)} <= seen
    assert {("whole", s) for s in (16, 32, 48)} <= seen
    assert {"first", "middle", "last", "long", "16 bytes", "empty off grid", "throw before a partial"} <= seen, seen


@pytest.mark.parametrize("model", [O.MODEL_COUNTER, O.MODEL_BANK_ACCOUNT], ids=["counter", "bank_account"])
def test_granular_logs_match_the_sample_model_oracle(model):
    """A third witness: the port of the reference fold walks each segment by byte offset and throws on a short tail
    (decode_event), so on 16-byte-granular logs it equals the program oracle for the Counter and BankAccount."""
    rng = np.random.default_rng(38000 + model)
    prog = P.counter_program() if model == O.MODEL_COUNTER else P.bank_account_program()
    rules, sb = rules_of(prog), int(prog.state_bytes)
    f64 = [int(prog.f64_field_off[i]) for i in range(prog.n_f64_fields)]
    counts = rng.integers(0, 10, size=40_000)
    counts[17] = 3000
    n = int(counts.sum())
    rec = rng.integers(0, 256, size=(n, 64), dtype=np.uint8)
    types = rng.integers(0, 2, size=n).astype(np.uint32)
    types[rng.random(n) < 0.001] = 2 if model == O.MODEL_BANK_ACCOUNT else 7   # scala.MatchError
    rec[:, 0:4] = types.view(np.uint8).reshape(-1, 4)
    if model == O.MODEL_BANK_ACCOUNT:
        rec[:, 32:40] = np.asarray(PC.SPECIAL_F64)[rng.integers(0, len(PC.SPECIAL_F64), size=n)].view(np.uint8).reshape(-1, 8)
    tails = np.where(rng.random(len(counts)) < 0.05, 16 * rng.integers(1, 4, size=len(counts)), 0)
    tails[[0, 17, len(counts) - 1]] = [16, 32, 48]
    for start in (16, 32, 48, 64 + 16):
        log, seg = PC.granular_log(rng, rec, counts, tails, start)
        want, nev, nerr = O.fold_packed(model, O.REC_FIXED64, log, seg)
        got, gev, gerr = I.c_fold(rules, sb, log[start:], seg, f64_fields=f64)
        same(got, want, f"model {model} start {start}")
        assert (gev, gerr) == (nev, nerr) and nerr > int((tails > 0).sum()) // 2, f"model {model} start {start}"
        want2, nev2, nerr2 = O.fold_packed(model, O.REC_FIXED64, log, seg, want)
        got2, gev2, gerr2 = I.c_fold(rules, sb, log[start:], seg, initial=want, f64_fields=f64)
        same(got2, want2, f"model {model} start {start} with prior states")
        assert (gev2, gerr2) == (nev2, nerr2)


@pytest.mark.parametrize("seed", range(60))
def test_arrival_order_matches_the_interpreter(seed):
    """Micro-batches onto a live table (per-batch flags cleared, untouched slots kept), and the from-None form."""
    rng = np.random.default_rng(32000 + seed)
    state_bytes, rules, f64 = PC.draw_program(rng)
    n_agg = 80
    rec, off, aggs = PC.draw_log(rng, len(rules), n_agg, 100, f64)
    perm = PC.interleave(rng, aggs)
    want = I.fold(rules, state_bytes, rec, off, f64_fields=f64)
    got, _, _ = I.c_fold_arrival_order(rules, state_bytes, rec[perm], None, f64_fields=f64, n_agg=n_agg)
    what = f"seed {seed} state_bytes {state_bytes} rules {rules} f64 {f64}"
    same(got, want, what + " from None")
    table = want
    for b in range(3):
        recb, _, aggb = PC.draw_log(rng, len(rules), n_agg, [30, 5, 200][b], f64)
        keep = rng.random(len(recb)) < 0.6                    # not every aggregate is touched
        batch = recb[PC.interleave(rng, aggb)][keep[: len(recb)]]
        want_b = I.fold_arrival_order(rules, state_bytes, batch, table, f64_fields=f64)
        got_b, nev, nerr = I.c_fold_arrival_order(rules, state_bytes, batch, table, f64_fields=f64)
        same(got_b, want_b, f"{what} batch {b}")
        touched = np.bincount(batch[:, 8:16].copy().view(np.uint64).ravel().astype(np.int64), minlength=n_agg)
        assert (nev, nerr) == implied_stats(want_b, state_bytes, touched), what
        table = want_b
    bad = rec[:3].copy()
    bad[1, 8:16] = np.frombuffer(np.uint64(n_agg).tobytes(), np.uint8)
    with pytest.raises(ValueError):
        I.c_fold_arrival_order(rules, state_bytes, bad, table, f64_fields=f64)


@pytest.mark.parametrize("max_record_bytes", [528, 1040, 2064])
@pytest.mark.parametrize("seed", range(30))
def test_variable_records_match_the_interpreter(seed, max_record_bytes):
    """SGR_REC_VAR16 logs with short, overlong and truncated records, from None and with prior states, under each cap."""
    rng = np.random.default_rng(33000 + seed)
    state_bytes, rules = PC.draw_var_program(rng)
    counts = rng.integers(0, 8, size=70)
    counts[int(rng.integers(0, 70))] = 120
    buf, seg, _ = PC.var_log(rng, rules, counts, max_record_bytes - 16 + 32, p_short=0.05, p_throw=0.01, n_malformed=3)
    what = f"seed {seed} cap {max_record_bytes} state_bytes {state_bytes} rules {rules}"
    want = I.fold_var(rules, state_bytes, buf, seg, max_record_bytes=max_record_bytes)
    got, nev, nerr = I.c_fold_var(rules, state_bytes, buf, seg, max_record_bytes=max_record_bytes)
    same(got, want, what)
    t = want.reshape(-1, state_bytes)
    assert nerr == int(((t[:, state_bytes - 8] & I.ST_ERROR) != 0).sum()), what
    want2 = I.fold_var(rules, state_bytes, buf, seg, initial=want, max_record_bytes=max_record_bytes)
    got2, _, _ = I.c_fold_var(rules, state_bytes, buf, seg, initial=want, max_record_bytes=max_record_bytes)
    same(got2, want2, what + " with prior states")


def test_the_draws_cover_what_the_pin_claims():
    """The random programs above reach every state width, the 64-bit ops, Double fields and every exists rule."""
    widths, ops, f64s, rules_seen = set(), set(), 0, set()
    for seed in range(160):
        state_bytes, rules, f64 = PC.draw_program(np.random.default_rng(31000 + seed))
        widths.add(state_bytes); f64s += bool(f64)
        for ex, tops in rules:
            rules_seen.add(ex); ops.update(o[0] for o in tops)
    assert widths == {16, 32, 48, 64, 128}
    assert ops == {I.OP_SET, I.OP_ADD_I32, I.OP_SUB_I32, I.OP_ADD_I64, I.OP_SUB_I64}
    assert rules_seen == {I.IF_EXISTS, I.MATERIALISE, I.CREATE, I.TOMBSTONE, I.THROW}
    assert f64s >= 20


def draw_wide_case(seed):
    """One wide variable-record program per seed (oracle/program_corpus.py draw_var_program_wide), the caps in turn, and
    a log whose record lengths sit around the cap (tests/test_gpu_var_limits.py folds the same kind of case)."""
    rng = np.random.default_rng(36000 + seed)
    cap = PC.VAR_CAPS[seed % len(PC.VAR_CAPS)]
    state_bytes, rules, f64 = PC.draw_var_program_wide(rng, cap)
    counts = rng.integers(0, 7, size=50)
    counts[int(rng.integers(0, 50))] = 60
    buf, seg, _ = PC.var_log_of(rng, rules, counts, PC.cap_lengths(rng, int(counts.sum()), cap), p_throw=0.01,
                                f64_srcs=(16, 24, 32))
    return rng, cap, state_bytes, rules, f64, counts, buf, seg


@pytest.mark.parametrize("seed", range(240))
def test_wide_variable_programs_match_the_interpreter(seed):
    """Every state width, 64-bit ops at 4-aligned destinations, long SETs, Double fields, sources up to the cap, records
    on both sides of it: the compiled oracle equals the interpreter, from None and on top of the first table."""
    rng, cap, state_bytes, rules, f64, counts, buf, seg = draw_wide_case(seed)
    what = f"seed {seed} cap {cap} state_bytes {state_bytes} rules {rules} f64 {f64}"
    want = I.fold_var(rules, state_bytes, buf, seg, f64_fields=f64, max_record_bytes=cap)
    got, nev, nerr = I.c_fold_var(rules, state_bytes, buf, seg, f64_fields=f64, max_record_bytes=cap)
    same(got, want, what)
    assert (nev, nerr) == implied_stats(want, state_bytes, counts), what
    want2 = I.fold_var(rules, state_bytes, buf, seg, initial=want, f64_fields=f64, max_record_bytes=cap)
    got2, nev2, nerr2 = I.c_fold_var(rules, state_bytes, buf, seg, initial=want, f64_fields=f64, max_record_bytes=cap)
    same(got2, want2, what + " with prior states")
    assert (nev2, nerr2) == implied_stats(want2, state_bytes, counts), what


def test_the_wide_draws_cover_what_the_pin_claims():
    """The wide draws reach every state width 16..128, class 0 / class 1 / mixed programs, 16 types, 8 ops, SETs of 48
    bytes and more, 64-bit ops at destinations = 4 (mod 8), a Double in the last 8 bytes of the program area, sources
    within 16 bytes of the cap, and records one byte under, at and one byte over the cap."""
    seen = set()
    for seed in range(240):
        _, cap, state_bytes, rules, f64, _, _, _ = draw_wide_case(seed)
        seen.add(("width", state_bytes))
        kinds = {ex for ex, _ in rules}
        seen.add("class1" if I.MATERIALISE not in kinds and I.IF_EXISTS in kinds else "mixed" if {I.MATERIALISE, I.IF_EXISTS} <= kinds
                 else "class0" if I.IF_EXISTS not in kinds else None)
        seen.add(("types", len(rules)))
        if state_bytes - 16 in f64:                       # user - 8: the last 8 bytes of the program area
            seen.add("f64 last")
        for _, ops in rules:
            seen.add(("ops", len(ops)))
            for opc, dst, src, ln in ops:
                if opc == I.OP_SET and ln >= 48:
                    seen.add("set48")
                if opc >= I.OP_ADD_I64 and dst % 8 == 4:
                    seen.add("i64 at 4 mod 8")
                if src + ln > cap - 16:
                    seen.add("src near cap")
    assert {("width", w) for w in range(16, 129, 16)} <= seen, sorted(x for x in seen if isinstance(x, tuple) and x[0] == "width")
    assert {"class0", "class1", "mixed"} <= seen
    assert ("types", 16) in seen and ("ops", 8) in seen
    assert {"set48", "i64 at 4 mod 8", "f64 last", "src near cap"} <= seen
    rng = np.random.default_rng(7)
    for cap in PC.VAR_CAPS:
        lens = PC.cap_lengths(rng, 4000, cap)
        assert {cap - 1, cap, cap + 1} <= set(lens.tolist()) and lens.max() > 2064, cap


SAMPLE_MODELS = [("counter", O.MODEL_COUNTER, P.counter_program), ("ml_counter", O.MODEL_ML_COUNTER, P.ml_counter_program),
                 ("int_balance", O.MODEL_INT_BALANCE, P.int_balance_program), ("bank_account", O.MODEL_BANK_ACCOUNT, P.bank_account_program)]


@pytest.mark.parametrize("name,model,make", SAMPLE_MODELS, ids=[m[0] for m in SAMPLE_MODELS])
def test_sample_programs_match_the_sample_model_oracle(name, model, make):
    """The four sample programs through the program oracle equal the hand-written Scala restatement, over 10^6 events
    with throws, MatchErrors and (BankAccount) special Doubles, from None and on top of the first table."""
    rng = np.random.default_rng(34000 + model)
    prog = make()
    rules, sb = rules_of(prog), int(prog.state_bytes)
    f64 = [int(prog.f64_field_off[i]) for i in range(prog.n_f64_fields)]
    counts = rng.integers(1, 10, size=250_000)
    counts[17] = 20_000
    counts[rng.integers(0, len(counts), size=30_000)] = 0
    if model == O.MODEL_BANK_ACCOUNT:
        n = int(counts.sum())
        rec = rng.integers(0, 256, size=(n, 64), dtype=np.uint8)
        types = np.where(rng.random(n) < 0.3, 0, 1).astype(np.uint32)
        types[rng.random(n) < 0.001] = 2                                       # scala.MatchError
        rec[:, 0:4] = types.view(np.uint8).reshape(-1, 4)
        rec[:, 8:16] = np.repeat(np.arange(len(counts), dtype=np.uint64), counts).view(np.uint8).reshape(-1, 8)
        rec[:, 32:40] = np.asarray(PC.SPECIAL_F64)[rng.integers(0, len(PC.SPECIAL_F64), size=n)].view(np.uint8).reshape(-1, 8)
        off = np.zeros(len(counts) + 1, np.uint64)
        np.cumsum(counts * 64, out=off[1:])
    else:
        rec, off = S.counter_csr(len(counts), counts, seed=71 + model, p_throw=0.0005)
        if model == O.MODEL_INT_BALANCE:
            rec = rec.copy()
            rec["type"] = np.where(rng.random(len(rec)) < 0.001, 1, 0)        # type 1 is a MatchError for IntBalance
    assert int(off[-1]) // 64 >= 1_000_000
    want, nev, nerr = O.fold_packed(model, O.REC_FIXED64, rec, off)
    got, gev, gerr = I.c_fold(rules, sb, rec, off, f64_fields=f64)
    same(got, want, name)
    assert (gev, gerr) == (nev, nerr) and nerr > 0, name
    want2, nev2, nerr2 = O.fold_packed(model, O.REC_FIXED64, rec, off, want)
    got2, gev2, gerr2 = I.c_fold(rules, sb, rec, off, initial=want, f64_fields=f64)
    same(got2, want2, name + " with prior states")
    assert (gev2, gerr2) == (nev2, nerr2), name


# ------------------------------------------------------------------ sort-free programs (the bulk fold and the routed path)
def draw_sort_free_case(seed):
    """One drawn sort-free program per seed, cycling through the four layouts, with and without tombstones, and 1..14 sources."""
    rng = np.random.default_rng(35000 + seed)
    layout = PC.LAYOUTS[seed % 4]
    tomb = layout == ("set", "set") and (seed // 4) % 2 == 1
    n_src = 1 + seed % 6 if seed % 10 else int(rng.integers(7, 15))
    rules, n_slots = PC.draw_sort_free_program(rng, layout=layout, tombstones=tomb, n_src=n_src)
    return rng, layout, tomb, rules, n_slots


@pytest.mark.parametrize("seed", range(300))
def test_sort_free_programs_have_their_layout_and_match_the_interpreter(seed):
    rng, layout, tomb, rules, n_slots = draw_sort_free_case(seed)
    lay = PC.bulk_layout(rules)
    what = f"seed {seed} layout {layout} tombstones {tomb} rules {rules}"
    assert lay is not None, what
    assert lay["set_only_mask"] == sum(1 << w for w in range(2) if layout[w] == "set"), what
    assert lay["has_none"] == int(tomb), what
    assert PC.row_slots(rules) == n_slots, what
    rec, off, _ = PC.draw_sort_free_log(rng, rules, 60, 400, 150, p_throw=0.02)
    want = I.fold(rules, 16, rec, off)
    got, nev, nerr = I.c_fold(rules, 16, rec, off)
    same(got, want, what)
    assert (nev, nerr) == implied_stats(want, 16, np.diff(off.astype(np.int64)) // 64), what


def test_bulk_layout_twin_on_known_programs():
    """bulk_fold.cu bulk_layout_for by hand: the Counter (add, set), the snapshot restore (set, set) with tombstones, and
    programs outside the class (a word both set and added, IF_EXISTS, a 32-byte state, a 64-bit add)."""
    counter = rules_of(P.counter_program())
    assert PC.bulk_layout(counter) == dict(set_only_mask=2, has_none=0, entry_shift=4, word_off=[4, 8], last_needed_mask=0b0100)
    restore = [(I.CREATE, [(I.OP_SET, 0, 16, 4), (I.OP_SET, 4, 20, 4)]), (I.TOMBSTONE, [])]
    assert PC.bulk_layout(restore) == dict(set_only_mask=3, has_none=1, entry_shift=5, word_off=[8, 16], last_needed_mask=0b11)
    set_add = [(I.MATERIALISE, [(I.OP_SET, 0, 4, 4), (I.OP_ADD_I32, 4, 16, 4)]), (I.MATERIALISE, []), (I.THROW, [])]
    assert PC.bulk_layout(set_add) == dict(set_only_mask=1, has_none=0, entry_shift=4, word_off=[8, 4], last_needed_mask=0b10)
    assert PC.bulk_layout([(I.MATERIALISE, [(I.OP_SET, 0, 16, 4)]), (I.MATERIALISE, [(I.OP_ADD_I32, 0, 20, 4)])]) is None
    assert PC.bulk_layout([(I.IF_EXISTS, [(I.OP_SET, 0, 16, 4)])]) is None
    assert PC.bulk_layout([(I.MATERIALISE, [(I.OP_SET, 0, 16, 4)])], state_bytes=32) is None
    assert PC.bulk_layout([(I.MATERIALISE, [(I.OP_ADD_I64, 0, 16, 8)])]) is None
    assert PC.bulk_layout([(I.MATERIALISE, [(I.OP_SET, 0, 16, 4), (I.OP_SET, 0, 20, 4)])]) is None   # a word written twice


def test_the_sort_free_draws_cover_what_the_routed_tests_claim():
    """The draws reach every layout with and without tombstones, rules without ops, SUB, 1..16 types, 2..7 slots and 8 or
    more, and reads of the type word, seq, bytes 16..31 and bytes 32..63; the log carries ADDs of 0 and every MatchError."""
    seen = set()
    for seed in range(300):
        _, layout, tomb, rules, n_slots = draw_sort_free_case(seed)
        seen.add((layout, tomb))
        seen.add(("types", len(rules)))
        seen.add(("slots", min(n_slots, 8)))
        for ex, ops in rules:
            if ex in (I.MATERIALISE, I.CREATE) and not ops:
                seen.add("no ops")
            for opc, _, src, _ in ops:
                seen.add("sub" if opc == I.OP_SUB_I32 else "op")
                seen.add(("read", 0 if src == 0 else 1 if src == 4 else 16 if src < 32 else 32))
    for layout in PC.LAYOUTS:
        assert (layout, False) in seen
    assert (("set", "set"), True) in seen
    assert {("types", k) for k in range(1, 17)} <= seen, sorted(x for x in seen if x[0] == "types")
    assert {("slots", k) for k in range(2, 9)} <= seen
    assert {"no ops", "sub", ("read", 0), ("read", 1), ("read", 16), ("read", 32)} <= seen
    rng = np.random.default_rng(5)
    rules, _ = PC.draw_sort_free_program(rng, layout=("add", "add"), n_types=3)
    rec, off, hot = PC.draw_sort_free_log(rng, rules, 100, 20_000, 4096, p_throw=0.05)
    types = rec[:, 0:4].copy().view(np.uint32).ravel()
    assert set(range(3, 16)) | set(PC.FAR_TYPES) <= set(types.tolist())
    assert (rec[:, 16:20].copy().view(np.uint32) == 0).any()
    assert int(off[hot + 1] - off[hot]) // 64 == 4096
    assert (np.diff(off.astype(np.int64)) == 0).any()
    rec0, _, _ = PC.draw_sort_free_log(rng, rules, 100, 20_000, 10, p_throw=0.0)
    assert (rec0[:, 0:4].copy().view(np.uint32) < 3).all()

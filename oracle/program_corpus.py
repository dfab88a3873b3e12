"""TEST INFRASTRUCTURE — random fold programs and logs for the program tests (tests/test_gpu_program_fuzz.py,
tests/test_gpu_program_scale.py, tests/test_gpu_var_limits.py, tests/test_gpu_fixed_alignment.py,
tests/test_program_oracle_cpu.py).

draw_program / draw_log / interleave / draw_var_program / draw_var_log are the small-case drawers of the fuzz test, moved
here unchanged: the same seeds give byte-identical programs and logs. The scale drawers below build logs of millions of
records whose shape (segment lengths, hot aggregate, empty runs, throws) is chosen by the caller, with numpy only.
"""
from __future__ import annotations

import numpy as np

from oracle import program_interp as I

SPECIAL_F64 = [0.0, -0.0, float("nan"), 1.5, float("inf"), -2.25]


def draw_program(rng):
    state_bytes = int(rng.choice([16, 32, 64, 48, 128], p=[0.35, 0.25, 0.2, 0.1, 0.1]))
    user = state_bytes - 8
    family = rng.choice(["class0", "class1", "mixed"], p=[0.45, 0.35, 0.2])
    pool = {"class0": [I.MATERIALISE, I.CREATE, I.TOMBSTONE, I.THROW], "class1": [I.IF_EXISTS, I.CREATE, I.TOMBSTONE, I.THROW],
            "mixed": [I.IF_EXISTS, I.MATERIALISE, I.CREATE, I.TOMBSTONE, I.THROW]}[family]
    weights = {4: [0.55, 0.25, 0.1, 0.1], 5: [0.3, 0.3, 0.2, 0.1, 0.1]}[len(pool)]
    wide_ops = rng.random() < 0.15
    n_types = int(rng.integers(1, 7))
    rules = []
    for t in range(n_types):
        ex = int(rng.choice(pool, p=weights)) if t else int(pool[0] if rng.random() < 0.5 else pool[1])   # type 0 creates something
        ops = []
        for _ in range(int(rng.integers(0, 5))):
            opc = int(rng.choice([I.OP_SET, I.OP_ADD_I32, I.OP_SUB_I32])) if not wide_ops else int(rng.integers(0, 5))
            ln = 4 if opc in (I.OP_ADD_I32, I.OP_SUB_I32) else 8 if opc in (I.OP_ADD_I64, I.OP_SUB_I64) else int(rng.choice([4, 8, 12, 16]))
            ln = min(ln, user)
            if opc in (I.OP_ADD_I64, I.OP_SUB_I64) and user < 8:
                continue
            dst = 4 * int(rng.integers(0, (user - ln) // 4 + 1))
            src = 4 if rng.random() < 0.2 and ln == 4 else 16 + 4 * int(rng.integers(0, (48 - ln) // 4 + 1))
            ops.append((opc, dst, src, ln))
        rules.append((ex, ops))
    f64 = []
    if user >= 16 and rng.random() < 0.4:
        off = 8 * int(rng.integers(0, user // 8))
        f64 = [off]
        # make sure some rule copies a double into that field, from an 8-aligned payload offset
        t = int(rng.integers(0, n_types))
        if rules[t][0] not in (I.TOMBSTONE, I.THROW):
            rules[t] = (rules[t][0], list(rules[t][1])[:3] + [(I.OP_SET, off, 24, 8)])
    return state_bytes, rules, f64


# ------------------------------------------------------------------ sort-free programs (bulk_fold.cu, route_push.cu)
# The four bulk entry layouts by (mode of state word 0, mode of state word 1). CREATE and TOMBSTONE reset both words, which
# makes both set words (fold_rows.cu build_row_program), so tombstones and CREATE come only with ("set", "set").
LAYOUTS = [("add", "add"), ("add", "set"), ("set", "add"), ("set", "set")]
# record words a sort-free program may read: the type word, seq, and the payload words 4..15 (bytes 16..63); words 2 and 3
# hold the aggregate index
SORT_FREE_SOURCES = [0, 1] + list(range(4, 16))


def draw_sort_free_program(rng, layout=None, tombstones=None, n_types=None, n_src=None):
    """A 16-byte class-0 program in which each state word is add-only or set-only: MATERIALISE / CREATE / TOMBSTONE / THROW
    rules, 32-bit ops only. layout: one of LAYOUTS; tombstones: only with ("set", "set"); n_types: 1..16 (raised to fit the
    sources); n_src: distinct record words read, 1..14 (n_slots = 1 + n_src: 2..7 fit a compact exchange record, 8 and more
    do not). Returns (rules, n_slots)."""
    layout = tuple(layout) if layout is not None else LAYOUTS[int(rng.integers(0, 4))]
    both_set = layout == ("set", "set")
    if tombstones is None:
        tombstones = both_set and rng.random() < 0.5
    assert both_set or not tombstones, "a tombstone resets both words: only the (set, set) layout has tombstones"
    n_src = int(rng.integers(1, 7)) if n_src is None else int(n_src)
    pool = [int(w) for w in rng.choice(SORT_FREE_SOURCES, size=n_src, replace=False)]
    todo = list(pool)
    n_op_rules = -(-n_src // 2)
    n_types = int(rng.integers(1, 17)) if n_types is None else int(n_types)
    n_types = min(16, max(n_types, n_op_rules + int(tombstones)))
    writers = [I.MATERIALISE, I.CREATE] if both_set else [I.MATERIALISE]
    extra = writers + [I.MATERIALISE, I.THROW] + ([I.TOMBSTONE] if tombstones else [])

    def op(word, ex):
        src = todo.pop() if todo else int(rng.choice(pool))
        if layout[word] == "add":
            opc = int(rng.choice([I.OP_ADD_I32, I.OP_SUB_I32]))
        else:   # over a reset state (CREATE) an ADD or a SUB is a set too
            opc = int(rng.choice([I.OP_SET, I.OP_ADD_I32, I.OP_SUB_I32])) if ex == I.CREATE else I.OP_SET
        return (opc, 4 * int(word), 4 * src, 4)

    rules = []
    for t in range(n_types):
        if t < n_op_rules:   # these rules read every source once and write both words, so the layout is what was asked
            ex = int(rng.choice(writers))
            ops = [op(w, ex) for w in rng.permutation(2)]
        else:
            ex = int(rng.choice(extra))
            if t == n_op_rules and tombstones:
                ex = I.TOMBSTONE
            ops = [] if ex in (I.TOMBSTONE, I.THROW) else [op(int(w), ex) for w in rng.permutation(2)[:int(rng.integers(0, 3))]]
        rules.append((ex, ops))
    assert not todo
    order = rng.permutation(n_types)
    return [rules[int(i)] for i in order], 1 + n_src


def row_slots(rules):
    """n_slots of fold_rows.cu build_row_program for a program it accepts: slot 0 is the event type, then one slot per
    distinct record word the ops read (a read of the type word takes a slot of its own)."""
    words = set()
    for ex, ops in rules:
        if ex in (I.TOMBSTONE, I.THROW):
            continue
        for _, _, src, ln in ops:
            words.update(range(src // 4, (src + ln) // 4))
    return 1 + len(words)


def bulk_layout(rules, state_bytes=16):
    """Twin of bulk_fold.cu bulk_layout_for (after build_row_program): None when the program is outside the sort-free class,
    else dict(set_only_mask, has_none, entry_shift, word_off, last_needed_mask)."""
    if state_bytes != 16 or len(rules) > 16 or any(ex == I.IF_EXISTS for ex, _ in rules):
        return None
    has_add = has_set = has_none = 0
    sets_of = {}
    for t, (ex, ops) in enumerate(rules):
        if ex == I.THROW:
            continue
        reset = ex in (I.CREATE, I.TOMBSTONE)
        mode = [2, 2] if reset else [0, 0]
        written = [False, False]
        for opc, dst, src, ln in ([] if ex == I.TOMBSTONE else ops):
            if opc > I.OP_SUB_I32 or src + ln > 64:
                return None
            for j in range(ln // 4):
                w = dst // 4 + j
                if w >= 2 or written[w]:
                    return None
                written[w] = True
                mode[w] = 2 if (opc == I.OP_SET or reset) else 1
        if row_slots(rules) > 16:
            return None
        has_none |= ex == I.TOMBSTONE
        for w in range(2):
            has_add |= (mode[w] == 1) << w
            has_set |= (mode[w] == 2) << w
        sets_of[t] = 2 in mode
    if has_add & has_set:
        return None
    n_set = bin(has_set & 3).count("1")
    if n_set == 2:
        shift, word_off = 5, [8, 16]
    elif n_set == 1:
        ws = 0 if has_set & 1 else 1
        shift, word_off = 4, [0, 0]
        word_off[ws], word_off[ws ^ 1] = 8, 4
    else:
        shift, word_off = 4, [4, 8]
    last = 0
    for t, sets in sets_of.items():
        if has_none or not sets:
            last |= 1 << t
    return dict(set_only_mask=has_set, has_none=int(has_none), entry_shift=shift, word_off=word_off, last_needed_mask=last)


# MatchError types a routed log carries besides n_types..15: the projected record keeps min(type, 16) in 5 bits, so types of
# 32 and more are where a missing clamp would wrap into a valid type
FAR_TYPES = [16, 17, 32, 33, 48, 1 << 31, 0xFFFFFFFF]


def draw_sort_free_log(rng, rules, n_agg, n_rec, hot_len, p_throw=0.0, p_empty=0.1, p_zero=0.05):
    """Fixed records in CSR order over n_agg aggregates (about n_rec records, the aggregate index at +8): random payload
    words and a random seq (set values are not monotone along an aggregate), a share p_empty of empty aggregates, one hot
    aggregate of hot_len records, record words 4..15 zero with probability p_zero (ADDs of 0), and with probability p_throw a
    throwing type: a THROW rule or a MatchError (n_types..15 and FAR_TYPES). Returns (records [n, 64] u8, seg_offsets, hot)."""
    counts = rng.geometric(1.0 / (n_rec / n_agg + 1), size=n_agg) - 1
    counts[rng.random(n_agg) < p_empty] = 0
    hot = int(rng.integers(0, n_agg))
    counts[hot] = hot_len
    n = int(counts.sum())
    rec = rng.integers(0, 256, size=(n, 64), dtype=np.uint8)
    words = rec.view(np.uint32)
    zero = rng.random((n, 12)) < p_zero
    words[:, 4:16][zero] = 0
    ok = np.array([t for t, (ex, _) in enumerate(rules) if ex != I.THROW], dtype=np.uint32)
    bad = np.array([t for t, (ex, _) in enumerate(rules) if ex == I.THROW] + list(range(len(rules), 16)) + FAR_TYPES, dtype=np.uint32)
    types = ok[rng.integers(0, len(ok), size=n)] if len(ok) else bad[rng.integers(0, len(bad), size=n)]
    hit = rng.random(n) < p_throw
    types[hit] = bad[rng.integers(0, len(bad), size=int(hit.sum()))]
    words[:, 0] = types
    words[:, 2:4] = np.repeat(np.arange(n_agg, dtype=np.uint64), counts).view(np.uint32).reshape(-1, 2)
    off = np.zeros(n_agg + 1, dtype=np.uint64)
    np.cumsum(counts * 64, out=off[1:])
    return rec, off, hot


def draw_log(rng, n_types, n_agg, long_len, f64):
    counts = rng.integers(0, 13, size=n_agg)
    counts[rng.integers(0, n_agg)] = long_len
    counts[rng.integers(0, n_agg, size=n_agg // 10)] = 0
    n = int(counts.sum())
    rec = rng.integers(0, 256, size=(n, 64), dtype=np.uint8)
    types = rng.integers(0, n_types, size=n).astype(np.uint32)
    types[rng.random(n) < 0.004] = n_types                       # scala.MatchError
    rec[:, 0:4] = types.view(np.uint8).reshape(-1, 4)
    rec[:, 4:8] = np.arange(1, n + 1, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
    aggs = np.repeat(np.arange(n_agg, dtype=np.uint64), counts)
    rec[:, 8:16] = aggs.view(np.uint8).reshape(-1, 8)
    if f64:
        hit = rng.random(n) < 0.5
        vals = np.asarray(SPECIAL_F64)[rng.integers(0, len(SPECIAL_F64), size=n)]
        rec[hit, 24:32] = vals[hit].view(np.uint8).reshape(-1, 8)
    off = np.zeros(n_agg + 1, dtype=np.uint64)
    np.cumsum(counts * 64, out=off[1:])
    return rec, off, aggs


def interleave(rng, aggs):
    """A permutation that shuffles aggregates against each other but keeps every aggregate's records in order
    (what a Kafka partition log looks like). `aggs` is in CSR order (non-decreasing)."""
    t = rng.random(len(aggs))
    times = t[np.lexsort((t, aggs))]     # within each aggregate the arrival times ascend with the log position
    return np.argsort(times, kind="stable")


# ------------------------------------------------------------------ variable records (SGR_REC_VAR16)
def draw_var_program(rng):
    """Like draw_program, with payload reads up to 80 bytes into the record and 16/32-byte states more likely (the
    record-parallel variable-record kernel takes 16-byte class-0 programs, everything else the lane-sequential kernel)."""
    state_bytes = int(rng.choice([16, 32, 64], p=[0.6, 0.25, 0.15]))
    user = state_bytes - 8
    pool = [I.MATERIALISE, I.CREATE, I.TOMBSTONE, I.THROW] if rng.random() < 0.7 else [I.IF_EXISTS, I.CREATE, I.TOMBSTONE, I.THROW]
    rules = []
    for t in range(int(rng.integers(1, 6))):
        ex = int(rng.choice(pool, p=[0.6, 0.2, 0.1, 0.1])) if t else int(I.CREATE if pool[0] == I.IF_EXISTS else pool[int(rng.integers(0, 2))])
        ops = []
        for _ in range(int(rng.integers(0, 4))):
            opc = int(rng.choice([I.OP_SET, I.OP_ADD_I32, I.OP_SUB_I32]))
            ln = 4 if opc != I.OP_SET else min(int(rng.choice([4, 8])), user)
            dst = 4 * int(rng.integers(0, (user - ln) // 4 + 1))
            src = 4 if rng.random() < 0.2 and ln == 4 else 16 + 4 * int(rng.integers(0, (80 - ln) // 4 + 1))
            ops.append((opc, dst, src, ln))
        rules.append((ex, ops))
    return state_bytes, rules


def draw_var_log(rng, n_types, n_agg, long_len):
    counts = rng.integers(0, 10, size=n_agg)
    counts[rng.integers(0, n_agg)] = long_len
    counts[rng.integers(0, n_agg, size=n_agg // 10)] = 0
    n = int(counts.sum())
    plen = rng.integers(80, 513, size=n)
    short = rng.random(n) < 0.03
    plen[short] = rng.integers(0, 80, size=int(short.sum()))          # too short for some event classes: those throw
    rlen = 16 + ((plen + 15) // 16) * 16
    rec_off = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(rlen, out=rec_off[1:])
    buf = rng.integers(0, 256, size=int(rec_off[-1]), dtype=np.uint8)
    types = rng.integers(0, n_types, size=n).astype(np.uint32)
    types[rng.random(n) < 0.004] = n_types
    aggs = np.repeat(np.arange(n_agg, dtype=np.uint32), counts)
    hdr = np.zeros((n, 4), dtype=np.uint32)
    hdr[:, 0], hdr[:, 1], hdr[:, 2], hdr[:, 3] = types, np.arange(1, n + 1, dtype=np.uint32), plen.astype(np.uint32), aggs
    hb = hdr.view(np.uint8).reshape(n, 16)
    starts = rec_off[:-1].astype(np.int64)
    for j in range(16):
        buf[starts + j] = hb[:, j]
    first = np.zeros(n_agg + 1, dtype=np.int64)
    np.cumsum(counts, out=first[1:])
    seg = rec_off[first].astype(np.uint64)
    # malformed records: a payload length that runs past the end of its segment (last record of a few segments), and one absurd one
    for a in rng.integers(0, n_agg, size=4):
        if counts[a]:
            j = int(first[a + 1] - 1)
            buf[int(rec_off[j]) + 8:int(rec_off[j]) + 12] = np.frombuffer(np.uint32(int(plen[j]) + 64).tobytes(), np.uint8)
    big = int(rng.integers(0, n))
    buf[int(rec_off[big]) + 8:int(rec_off[big]) + 12] = np.frombuffer(np.uint32(0x7FFFFFF0).tobytes(), np.uint8)
    return buf, seg, rec_off


VAR_CAPS = [64, 100, 520, 528, 529, 600, 1040, 1041, 1500, 2064]   # max_record_bytes values the variable-record tests use


def draw_var_program_wide(rng, cap, state_bytes=None):
    """A variable-record program over the whole language at record cap `cap` (max_record_bytes): every state width
    16..128, class 0 / class 1 / mixed rules, 1..16 types of 0..8 ops, SETs of any multiple of 4 that fits, 64-bit adds
    and subtracts at any 4-aligned destination, 0..2 Double fields (sometimes the last 8 bytes of the program area), and
    sources anywhere in [0, cap - len], a fifth of them within 16 bytes of the cap. cap = 64 draws a fixed-record program.
    Returns (state_bytes, rules, f64_fields)."""
    state_bytes = 16 * int(rng.integers(1, 9)) if state_bytes is None else int(state_bytes)
    user = state_bytes - 8
    family = ["class0", "class1", "mixed"][int(rng.integers(0, 3))]
    pool = {"class0": [I.MATERIALISE, I.CREATE, I.TOMBSTONE, I.THROW], "class1": [I.IF_EXISTS, I.CREATE, I.TOMBSTONE, I.THROW],
            "mixed": [I.IF_EXISTS, I.MATERIALISE, I.CREATE, I.TOMBSTONE, I.THROW]}[family]
    weights = {4: [0.55, 0.25, 0.1, 0.1], 5: [0.3, 0.3, 0.2, 0.1, 0.1]}[len(pool)]
    n_types = int(rng.integers(1, 17))
    rules = []
    for t in range(n_types):
        if t == 0:      # type 0 builds a state
            ex = I.CREATE if family == "class1" else [I.MATERIALISE, I.CREATE][int(rng.integers(0, 2))]
        elif family == "mixed" and t == 1:
            ex = I.IF_EXISTS
        else:
            ex = int(rng.choice(pool, p=weights))
        ops = []
        for _ in range(int(rng.integers(0, 9)) if ex not in (I.TOMBSTONE, I.THROW) else 0):
            opc = int(rng.choice([I.OP_SET, I.OP_ADD_I32, I.OP_SUB_I32, I.OP_ADD_I64, I.OP_SUB_I64], p=[0.4, 0.15, 0.15, 0.15, 0.15]))
            if opc >= I.OP_ADD_I64 and user < 8:
                opc = I.OP_SET
            if opc == I.OP_SET:
                ln = 4 * int(rng.integers(1, min(user, cap) // 4 + 1)) if rng.random() < 0.5 else 4 * int(rng.integers(1, 3))
            else:
                ln = 4 if opc <= I.OP_SUB_I32 else 8
            dst = 4 * int(rng.integers(0, (user - ln) // 4 + 1))
            top = (cap - ln) // 4                      # the last 4-aligned source that fits below the cap
            r = rng.random()
            if r < 0.2:
                src = 4 * int(rng.integers(max(0, top - 3), top + 1))
            elif r < 0.3:
                src = 4 * int(rng.integers(0, min(4, top + 1)))   # header words
            else:
                src = 4 * int(rng.integers(min(4, top), min(top, 4 + 24) + 1))
            ops.append((opc, dst, src, ln))
        rules.append((ex, ops))
    f64 = []
    if user >= 8 and rng.random() < 0.45:
        f64 = [user - 8] if rng.random() < 0.4 else [4 * int(rng.integers(0, (user - 8) // 4 + 1))]
        if user >= 24 and rng.random() < 0.5:
            other = [o for o in range(0, user - 7, 4) if abs(o - f64[0]) >= 8]
            f64.append(int(rng.choice(other)))
        t = int(rng.integers(0, n_types))               # some rule copies a Double into the first field
        if rules[t][0] not in (I.TOMBSTONE, I.THROW) and len(rules[t][1]) < 8:
            rules[t] = (rules[t][0], list(rules[t][1]) + [(I.OP_SET, f64[0], 16 + 8 * int(rng.integers(0, 3)), 8)])
    return state_bytes, rules, f64


def cap_lengths(rng, n, cap, ring=2064):
    """n record lengths (16 + payload_len, before padding) around the cap: a third anywhere in [16, cap], a third within
    16 bytes of the cap on either side, a third past it, up to 32 bytes past `ring` (a kernel's ring capacity)."""
    pick = rng.random(n)
    below = rng.integers(16, cap + 1, size=n)
    near = rng.integers(max(16, cap - 16), cap + 17, size=n)
    past = rng.integers(cap + 1, max(cap + 2, ring + 33), size=n)
    return np.where(pick < 1 / 3, below, np.where(pick < 2 / 3, near, past))


def var_log_of(rng, rules, counts, rec_bytes, p_throw=2e-4, f64_srcs=(), f64_values=SPECIAL_F64):
    """Variable records in CSR order with the given lengths (rec_bytes[i] = 16 + payload_len of record i, every record
    well formed and inside its segment), random payloads, types from type_mix, seq = position, the aggregate at +12.
    f64_srcs: record byte offsets that get values drawn from f64_values where the record holds them.
    Returns (log u8, seg_offsets u64, rec_offsets u64)."""
    n = int(counts.sum())
    plen = np.asarray(rec_bytes, dtype=np.int64) - 16
    assert len(plen) == n and (plen >= 0).all()
    rlen = 16 + ((plen + 15) // 16) * 16
    rec_off = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(rlen, out=rec_off[1:])
    buf = rng.integers(0, 256, size=int(rec_off[-1]), dtype=np.uint8)
    hdr = np.zeros((n, 4), dtype=np.uint32)
    hdr[:, 0] = type_mix(rules, n, rng, p_throw)
    hdr[:, 1] = np.arange(1, n + 1, dtype=np.uint32)
    hdr[:, 2] = plen.astype(np.uint32)
    hdr[:, 3] = np.repeat(np.arange(len(counts), dtype=np.uint32), counts)
    hb = hdr.view(np.uint8).reshape(n, 16)
    starts = rec_off[:-1].astype(np.int64)
    for j in range(16):
        buf[starts + j] = hb[:, j]
    vals = np.asarray(f64_values, dtype=np.float64)
    for src in f64_srcs:
        hit = np.nonzero(16 + plen >= src + 8)[0]
        vb = vals[rng.integers(0, len(vals), size=len(hit))].view(np.uint8).reshape(-1, 8)
        for j in range(8):
            buf[starts[hit] + src + j] = vb[:, j]
    first = np.zeros(len(counts) + 1, dtype=np.int64)
    np.cumsum(counts, out=first[1:])
    return buf, rec_off[first].astype(np.uint64), rec_off


# ------------------------------------------------------------------ scale: programs whose kernel instantiation is known
# Record words a row program may read: word 1 (seq) and the payload words 4..15 (words 2, 3 hold the aggregate index).
SOURCE_WORDS = [1] + list(range(4, 16))


def row_program(rng, user_words, cls, n_src):
    """A program inside the transformer algebra (fold_rows.cu build_row_program): 32-bit SET/ADD/SUB ops only, no rule
    writes a state word twice, and the ops read exactly `n_src` distinct record words, so the kernel sees
    n_slots = 1 + n_src (slot 0 is the event type). cls 0: MATERIALISE / CREATE / TOMBSTONE / THROW; cls 1: IF_EXISTS /
    CREATE / TOMBSTONE / THROW. Type 0 builds a state (MATERIALISE, or CREATE for class 1), type 1 carries the class."""
    pool = [int(w) for w in rng.choice(SOURCE_WORDS, size=n_src, replace=False)]
    base = I.MATERIALISE if cls == 0 else I.IF_EXISTS
    n_op_rules = -(-n_src // user_words) + 1
    n_types = min(16, n_op_rules + int(rng.integers(2, 5)))
    exists = [I.MATERIALISE if cls == 0 else I.CREATE, base]
    exists += [int(rng.choice([base, I.CREATE])) for _ in range(2, n_op_rules)]
    exists += [int(rng.choice([base, base, I.CREATE, I.TOMBSTONE, I.THROW])) for _ in range(n_op_rules, n_types)]
    todo = list(pool)
    rng.shuffle(todo)
    rules = []
    for t, ex in enumerate(exists):
        ops = []
        if ex not in (I.TOMBSTONE, I.THROW):
            dst_words = [int(w) for w in rng.permutation(user_words)]
            n_ops = min(user_words, 8, len(todo)) if t < n_op_rules else int(rng.integers(0, min(user_words, 4) + 1))
            n_ops = max(n_ops, min(user_words, 8, int(rng.integers(0, 3))))
            for w in dst_words[:n_ops]:
                src = todo.pop() if todo else int(rng.choice(pool))
                ops.append((int(rng.choice([I.OP_SET, I.OP_ADD_I32, I.OP_SUB_I32])), 4 * w, 4 * src, 4))
        rules.append((ex, ops))
    assert not todo
    return rules


# ------------------------------------------------------------------ named programs the fixed-record GPU tests share
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


# outside the transformer algebra: the lane-sequential kernel folds them
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


def type_mix(rules, n, rng, p_throw=2e-4):
    """Event types for n records: throwing types (THROW rules, MatchErrors at n_types .. 16, 255, 2^32 - 1) with
    probability p_throw, every other rule uniformly."""
    ok = np.array([t for t, (ex, _) in enumerate(rules) if ex != I.THROW], dtype=np.uint32)
    bad = np.array([t for t, (ex, _) in enumerate(rules) if ex == I.THROW] + list(range(len(rules), 17)) + [255, 0xFFFFFFFF],
                   dtype=np.uint32)
    types = ok[rng.integers(0, len(ok), size=n)]
    hit = rng.random(n) < p_throw
    types[hit] = bad[rng.integers(0, len(bad), size=int(hit.sum()))]
    return types


def shaped_counts(rng, n_agg, n_records, hot_share=0.25, step_records=256, empty_run=3000):
    """Segment lengths for a CSR of about n_records records: one hot aggregate holding hot_share of the log and a second
    one with a fifth of that, runs of `empty_run` empty segments at the start, the middle and the end, segments of exactly
    one step, and segments that start and end on step and span multiples (step_records: the longest run-kernel step,
    32 * 8 records). Returns (counts, hot, hot2)."""
    rest = n_records - int(n_records * hot_share)
    mean = rest / (n_agg - 3 * empty_run)
    counts = rng.geometric(1.0 / (mean + 1), size=n_agg) - 1
    counts[:empty_run] = 0
    mid = n_agg // 2
    counts[mid:mid + empty_run] = 0
    counts[-empty_run:] = 0
    hot, hot2 = empty_run + 1, n_agg - empty_run - 2
    counts[hot] = int(n_records * hot_share)
    counts[hot2] = int(n_records * hot_share / 5)
    # a few aligned segments: pad the prefix to a multiple of a step, then 1, 2, 8 and 64 steps
    for j, k in enumerate([1, 2, 8, 64, 1]):
        a = mid + empty_run + 10 + 40 * j
        pre = int(counts[:a].sum())
        counts[a] += (-pre) % step_records
        counts[a + 1] = k * step_records
    return counts.astype(np.int64), hot, hot2


def fixed_log(rng, rules, counts, f64_offsets=(), f64_values=SPECIAL_F64, pad_records=0, p_throw=2e-4):
    """Fixed 64-byte records in CSR order for per-aggregate `counts`: random payload, types from type_mix, seq = position,
    agg at +8. f64_offsets: record byte offsets that get values drawn from f64_values. pad_records: records in front of
    the first segment (the CSR starts at a non-zero offset). Returns (buffer [pad + n, 64] u8, seg_offsets u64, aggs)."""
    n = int(counts.sum())
    buf = rng.integers(0, 256, size=(pad_records + n, 64), dtype=np.uint8)
    rec = buf[pad_records:]
    rec[:, 0:4] = type_mix(rules, n, rng, p_throw).view(np.uint8).reshape(-1, 4)
    rec[:, 4:8] = np.arange(1, n + 1, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
    aggs = np.repeat(np.arange(len(counts), dtype=np.uint64), counts)
    rec[:, 8:16] = aggs.view(np.uint8).reshape(-1, 8)
    vals = np.asarray(f64_values, dtype=np.float64)
    for off in f64_offsets:
        rec[:, off:off + 8] = vals[rng.integers(0, len(vals), size=n)].view(np.uint8).reshape(-1, 8)
    seg = np.zeros(len(counts) + 1, dtype=np.uint64)
    np.cumsum(counts * 64, out=seg[1:])
    seg += pad_records * 64
    return buf, seg, aggs


def granular_log(rng, records, counts, tails, start):
    """Fixed records laid out at 16-byte granularity: `start` random bytes (a multiple of 16) in front of the first segment,
    then per aggregate counts[i] whole 64-byte records (records [n, 64] in CSR order) followed by tails[i] bytes (0, 16, 32
    or 48) of a trailing partial record whose first word is the valid type 0. Segment starts fall wherever the tails before
    them put them. Returns (log u8 flat, seg_offsets u64 byte offsets into the log)."""
    counts = np.asarray(counts, dtype=np.int64)
    tails = np.asarray(tails, dtype=np.int64)
    assert start % 16 == 0 and np.isin(tails, [0, 16, 32, 48]).all()
    rec = np.ascontiguousarray(records, dtype=np.uint8).reshape(-1, 64)
    n = int(counts.sum())
    assert len(rec) == n
    seg = np.zeros(len(counts) + 1, dtype=np.uint64)
    seg[0] = start
    seg[1:] = start + np.cumsum(64 * counts + tails)
    buf = rng.integers(0, 256, size=int(seg[-1]), dtype=np.uint8)
    units = buf.reshape(-1, 16)
    first = np.zeros(len(counts), dtype=np.int64)
    np.cumsum(counts[:-1], out=first[1:])
    at = np.repeat(seg[:-1].astype(np.int64) // 16 - 4 * first, counts) + 4 * np.arange(n, dtype=np.int64)
    units[at[:, None] + np.arange(4)] = rec.reshape(n, 4, 16)
    part = np.nonzero(tails)[0]
    buf[(seg[1:][part].astype(np.int64) - tails[part])[:, None] + np.arange(4)] = 0
    return buf, seg


def set_type(buf, seg, agg, k, etype):
    """Event type of record k of aggregate agg (k < 0 counts from the segment's end)."""
    rec = np.asarray(buf).reshape(-1, 64)
    lo, hi = int(seg[agg]) // 64, int(seg[agg + 1]) // 64
    rec[(lo if k >= 0 else hi) + k, 0:4] = np.frombuffer(np.uint32(etype).tobytes(), np.uint8)


def var_log(rng, rules, counts, payload_max, p_short=0.02, p_throw=2e-4, n_malformed=8):
    """Variable records (SGR_REC_VAR16) in CSR order: payload lengths uniform in [80, payload_max] (a few shorter than
    the ops of some event class read, which throw), a few records whose length runs past the end of their segment, and
    one absurd length. Returns (log u8, seg_offsets u64, rec_offsets u64) — rec_offsets is the record directory."""
    n = int(counts.sum())
    plen = rng.integers(80, payload_max + 1, size=n)
    short = rng.random(n) < p_short
    plen[short] = rng.integers(0, 80, size=int(short.sum()))
    plen[rng.integers(0, n, size=64)] = payload_max                     # at the cap, not past it
    rlen = 16 + ((plen + 15) // 16) * 16
    rec_off = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(rlen, out=rec_off[1:])
    buf = rng.integers(0, 256, size=int(rec_off[-1]), dtype=np.uint8)
    hdr = np.zeros((n, 4), dtype=np.uint32)
    hdr[:, 0] = type_mix(rules, n, rng, p_throw)
    hdr[:, 1] = np.arange(1, n + 1, dtype=np.uint32)
    hdr[:, 2] = plen.astype(np.uint32)
    hdr[:, 3] = np.repeat(np.arange(len(counts), dtype=np.uint32), counts)
    hb = hdr.view(np.uint8).reshape(n, 16)
    starts = rec_off[:-1].astype(np.int64)
    for j in range(16):
        buf[starts + j] = hb[:, j]
    first = np.zeros(len(counts) + 1, dtype=np.int64)
    np.cumsum(counts, out=first[1:])
    seg = rec_off[first].astype(np.uint64)
    for a in rng.choice(np.nonzero(counts)[0], size=n_malformed, replace=False):
        j = int(first[a + 1] - 1)
        buf[int(rec_off[j]) + 8:int(rec_off[j]) + 12] = np.frombuffer(np.uint32(int(plen[j]) + 64).tobytes(), np.uint8)
    big = int(rng.integers(0, n))
    buf[int(rec_off[big]) + 8:int(rec_off[big]) + 12] = np.frombuffer(np.uint32(0x7FFFFFF0).tobytes(), np.uint8)
    return buf, seg, rec_off

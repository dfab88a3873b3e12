"""TEST INFRASTRUCTURE — interpreter for arbitrary fold programs (include/sgr.h "fold program"), small cases only.

The fold-program language is this repository's declarative stand-in for AggregateCommandModel.handleEvent
(modules/command-engine/scaladsl/src/main/scala/surge/scaladsl/command/CommandModels.scala:14); the reference has no such
language, so this interpreter pins the CUDA kernels to the WRITTEN semantics of include/sgr.h, not to reference code.
What it takes from the reference are the rules around the fold, restated exactly as oracle/sgr_oracle.c does:
  events.foldLeft(state)(handleEvent)                      CommandModels.scala:25-28
  handler throws -> ACKError, the actor keeps its state    PersistentActor.scala:260-263,303-309
  publish iff newState != oldState (Double fields: ==)     PersistentActor.scala:252-257
Only tests/ may import it. One Python loop per event: use it on thousands of events, not millions. The c_* functions at
the end run the same semantics compiled (oracle/program_oracle.c) for logs of millions of records.
"""
from __future__ import annotations

import struct
from typing import Optional, Sequence, Tuple

import numpy as np

IF_EXISTS, MATERIALISE, CREATE, TOMBSTONE, THROW = range(5)
OP_SET, OP_ADD_I32, OP_SUB_I32, OP_ADD_I64, OP_SUB_I64 = range(5)
ST_EXISTS, ST_CHANGED, ST_ERROR = 1, 2, 4

Rule = Tuple[int, Sequence[Tuple[int, int, int, int]]]


class _Throw(Exception):
    pass


def _handle(rules: Sequence[Rule], user_bytes: int, state: Optional[bytearray], rec: bytes, avail: int = 64) -> Optional[bytearray]:
    """Returns the SAME object when the rule hands the instance back (no field op on an existing state: Scala `current`,
    `aggregate.map(identity)`), a NEW one when it builds or copies a state — object identity stands for JVM `eq`."""
    (etype,) = struct.unpack_from("<I", rec, 0)
    if etype >= len(rules):
        raise _Throw()                      # scala.MatchError
    exists_rule, ops = rules[etype]
    if exists_rule == THROW:
        raise _Throw()
    if exists_rule == TOMBSTONE:
        return None
    if any(src + ln > avail for _, _, src, ln in ops):
        raise _Throw()                      # the record is too short for this event class (variable records)
    if exists_rule == IF_EXISTS:
        if state is None:
            return None
        if not ops:
            return state
        cur = bytearray(state)
    elif exists_rule == MATERIALISE:
        if state is not None and not ops:
            return state
        cur = bytearray(state) if state is not None else bytearray(user_bytes)
    else:                                   # CREATE
        cur = bytearray(user_bytes)
    for opcode, dst, src, ln in ops:
        if opcode == OP_SET:
            cur[dst:dst + ln] = rec[src:src + ln]
        elif opcode in (OP_ADD_I32, OP_SUB_I32):
            a = struct.unpack_from("<I", cur, dst)[0]
            b = struct.unpack_from("<I", rec, src)[0]
            struct.pack_into("<I", cur, dst, (a + b if opcode == OP_ADD_I32 else a - b) & 0xFFFFFFFF)
        else:
            a = struct.unpack_from("<Q", cur, dst)[0]
            b = struct.unpack_from("<Q", rec, src)[0]
            struct.pack_into("<Q", cur, dst, (a + b if opcode == OP_ADD_I64 else a - b) & 0xFFFFFFFFFFFFFFFF)
    return cur


def _equal(a: Optional[bytearray], b: Optional[bytearray], f64_fields: Sequence[int]) -> bool:
    if (a is None) != (b is None):
        return False
    if a is None or a is b:                 # None == None; `this eq that`
        return True
    skip = set()
    for off in f64_fields:
        x = struct.unpack_from("<d", a, off)[0]
        y = struct.unpack_from("<d", b, off)[0]
        if not x == y:                      # JVM ==: 0.0 == -0.0, NaN != NaN
            return False
        skip.update(range(off, off + 8))
    return all(a[i] == b[i] for i in range(len(a)) if i not in skip)


def fold(rules: Sequence[Rule], state_bytes: int, records: np.ndarray, seg_offsets: Sequence[int], initial: Optional[np.ndarray] = None,
         f64_fields: Sequence[int] = ()) -> np.ndarray:
    """records: the log's bytes from seg_offsets[0] on ([n, 64] or flat uint8), in CSR order; seg_offsets: byte offsets
    (n_agg + 1), multiples of 16 apart. A segment's whole records fold at their own byte positions; a trailing 16, 32 or
    48 bytes is a malformed event, the handler throws there (include/sgr.h). Returns the state table [n_agg, state_bytes]."""
    user = state_bytes - 8
    buf = np.ascontiguousarray(records).view(np.uint8).reshape(-1).tobytes()
    n_agg = len(seg_offsets) - 1
    base = int(seg_offsets[0])
    out = np.zeros((n_agg, state_bytes), dtype=np.uint8)
    for i in range(n_agg):
        old: Optional[bytearray] = None
        if initial is not None:
            row = np.ascontiguousarray(initial).view(np.uint8).reshape(-1, state_bytes)[i]
            if struct.unpack_from("<I", row.tobytes(), user)[0] & ST_EXISTS:
                old = bytearray(row[:user].tobytes())
        cur = old                           # the actor's own instance
        pos, end, k, threw_at = int(seg_offsets[i]) - base, int(seg_offsets[i + 1]) - base, 0, -1
        assert pos % 16 == 0 and end % 16 == 0 and end >= pos, "segment offsets are 16-byte granular and monotone"
        while pos < end:
            try:
                if end - pos < 64:
                    raise _Throw()          # a trailing partial record
                cur = _handle(rules, user, cur, buf[pos:pos + 64])
            except _Throw:
                threw_at = k
                break
            pos += 64
            k += 1
        if threw_at >= 0:
            final, flags, err = old, ST_ERROR, threw_at
        else:
            final, flags, err = cur, (0 if _equal(old, cur, f64_fields) else ST_CHANGED), 0
        if final is not None:
            out[i, :user] = np.frombuffer(bytes(final), dtype=np.uint8)
            flags |= ST_EXISTS
        out[i, user:] = np.frombuffer(struct.pack("<II", flags, err), dtype=np.uint8)
    return out


def fold_arrival_order(rules: Sequence[Rule], state_bytes: int, records: np.ndarray, states: np.ndarray, f64_fields: Sequence[int] = ()) -> np.ndarray:
    """One micro-batch in arrival order onto a live table (records carry the aggregate index at +8): group stably by
    aggregate, then ApplyEvents per touched aggregate; untouched slots keep their state with the per-batch flags cleared."""
    recs = np.ascontiguousarray(records).view(np.uint8).reshape(-1, 64)
    table = np.ascontiguousarray(states).view(np.uint8).reshape(-1, state_bytes).copy()
    user = state_bytes - 8
    aggs = recs[:, 8:16].copy().view(np.uint64).ravel() if len(recs) else np.zeros(0, np.uint64)
    flags = table[:, user:user + 4].copy().view(np.uint32).ravel()
    table[:, user:user + 4] = (flags & ST_EXISTS).astype(np.uint32).view(np.uint8).reshape(-1, 4)
    table[:, user + 4:] = 0
    order = np.argsort(aggs, kind="stable")
    for a in np.unique(aggs):
        idx = order[np.searchsorted(aggs[order], a, "left"):np.searchsorted(aggs[order], a, "right")]
        seg = recs[idx]
        table[int(a)] = fold(rules, state_bytes, seg, [0, 64 * len(seg)], table[int(a):int(a) + 1], f64_fields)[0]
    return table


MAX_VAR_RECORD = 16 + 512   # include/sgr.h: a variable record is capped at 16 + 512 bytes unless "max_record_bytes" is raised


def fold_var(rules: Sequence[Rule], state_bytes: int, log: np.ndarray, seg_offsets: Sequence[int], initial: Optional[np.ndarray] = None,
             f64_fields: Sequence[int] = (), max_record_bytes: int = MAX_VAR_RECORD) -> np.ndarray:
    """Variable records (SGR_REC_VAR16): 16-byte header {type, seq, payload_len, agg} + payload padded to 16 bytes. A record
    that does not fit its segment, or is longer than the format allows (max_record_bytes, header included, before padding),
    or is too short for the ops of its event class, is a malformed event: the handler throws at that record, however much
    room a kernel's ring or stage would have had for it (tests/test_gpu_var_limits.py)."""
    user = state_bytes - 8
    buf = np.ascontiguousarray(log).view(np.uint8).reshape(-1).tobytes()
    n_agg = len(seg_offsets) - 1
    out = np.zeros((n_agg, state_bytes), dtype=np.uint8)
    for i in range(n_agg):
        old: Optional[bytearray] = None
        if initial is not None:
            row = np.ascontiguousarray(initial).view(np.uint8).reshape(-1, state_bytes)[i]
            if struct.unpack_from("<I", row.tobytes(), user)[0] & ST_EXISTS:
                old = bytearray(row[:user].tobytes())
        cur = old
        pos, end, k, threw_at = int(seg_offsets[i]), int(seg_offsets[i + 1]), 0, -1
        while pos < end:
            try:
                if end - pos < 16:
                    raise _Throw()
                plen = struct.unpack_from("<I", buf, pos + 8)[0]
                rlen = 16 + ((plen + 15) // 16) * 16
                if 16 + plen > max_record_bytes or rlen > end - pos:
                    raise _Throw()
                cur = _handle(rules, user, cur, buf[pos:pos + rlen], avail=16 + plen)
            except _Throw:
                threw_at = k
                break
            pos += rlen
            k += 1
        if threw_at >= 0:
            final, flags, err = old, ST_ERROR, threw_at
        else:
            final, flags, err = cur, (0 if _equal(old, cur, f64_fields) else ST_CHANGED), 0
        if final is not None:
            out[i, :user] = np.frombuffer(bytes(final), dtype=np.uint8)
            flags |= ST_EXISTS
        out[i, user:] = np.frombuffer(struct.pack("<II", flags, err), dtype=np.uint8)
    return out


# ------------------------------------------------------------------ the same semantics, compiled (oracle/program_oracle.c)
# Same argument shapes as the Python functions above; each also returns (n_events, n_errors): the events applied (those after
# a throw are dropped) and the aggregates whose handler threw. Use these at scale; tests/test_program_oracle_cpu.py pins
# them to the Python loops.

def _packed_program(rules: Sequence[Rule], state_bytes: int, f64_fields: Sequence[int]) -> np.ndarray:
    """orc_program of program_oracle.c: state_bytes, n_types, n_f64, f64_off[8], exists[16], n_ops[16], ops[16][8][4]."""
    p = np.zeros(3 + 8 + 16 + 16 + 16 * 8 * 4, dtype=np.uint32)
    p[0], p[1], p[2] = state_bytes, len(rules), len(f64_fields)
    p[3:3 + len(f64_fields)] = list(f64_fields)
    ops = p[43:].reshape(16, 8, 4)
    for t, (ex, tops) in enumerate(rules):
        p[11 + t] = ex
        p[27 + t] = len(tops)
        for i, op in enumerate(tops):
            ops[t, i] = op
    return p


def _lib():
    from oracle import oracle as O
    return O.lib()


def _ptr(a):
    return None if a is None else a.ctypes.data


def _prior(initial, n_agg, state_bytes):
    if initial is None:
        return None
    return np.ascontiguousarray(np.ascontiguousarray(initial).view(np.uint8).reshape(-1, state_bytes)[:n_agg])


def c_fold(rules: Sequence[Rule], state_bytes: int, records: np.ndarray, seg_offsets, initial: Optional[np.ndarray] = None,
           f64_fields: Sequence[int] = ()) -> Tuple[np.ndarray, int, int]:
    """fold(): `records` starts at byte seg_offsets[0]."""
    import ctypes as C
    prog = _packed_program(rules, state_bytes, f64_fields)
    recs = np.ascontiguousarray(records).view(np.uint8).reshape(-1)
    off = np.ascontiguousarray(seg_offsets, dtype=np.uint64)
    n_agg = len(off) - 1
    if int(off[-1]) - int(off[0]) > recs.size:
        raise ValueError("program oracle: CSR runs past the records")
    out = np.zeros((n_agg, state_bytes), dtype=np.uint8)
    ini = _prior(initial, n_agg, state_bytes)
    nev, nerr = C.c_uint64(0), C.c_uint64(0)
    if _lib().orc_prog_fold(_ptr(prog), _ptr(recs), _ptr(off), n_agg, _ptr(ini), _ptr(out), C.addressof(nev), C.addressof(nerr)):
        raise ValueError("program oracle: malformed program or CSR")
    return out, int(nev.value), int(nerr.value)


def c_fold_var(rules: Sequence[Rule], state_bytes: int, log: np.ndarray, seg_offsets, initial: Optional[np.ndarray] = None,
               f64_fields: Sequence[int] = (), max_record_bytes: int = MAX_VAR_RECORD) -> Tuple[np.ndarray, int, int]:
    """fold_var(): seg_offsets are byte offsets into the whole `log`."""
    import ctypes as C
    prog = _packed_program(rules, state_bytes, f64_fields)
    buf = np.ascontiguousarray(log).view(np.uint8).reshape(-1)
    off = np.ascontiguousarray(seg_offsets, dtype=np.uint64)
    n_agg = len(off) - 1
    if n_agg and int(off[-1]) > buf.size:
        raise ValueError("program oracle: CSR runs past the log")
    out = np.zeros((n_agg, state_bytes), dtype=np.uint8)
    ini = _prior(initial, n_agg, state_bytes)
    nev, nerr = C.c_uint64(0), C.c_uint64(0)
    if _lib().orc_prog_fold_var(_ptr(prog), max_record_bytes, _ptr(buf), _ptr(off), n_agg, _ptr(ini), _ptr(out),
                                C.addressof(nev), C.addressof(nerr)):
        raise ValueError("program oracle: malformed program or CSR")
    return out, int(nev.value), int(nerr.value)


def c_fold_arrival_order(rules: Sequence[Rule], state_bytes: int, records: np.ndarray, states: Optional[np.ndarray],
                         f64_fields: Sequence[int] = (), n_agg: Optional[int] = None) -> Tuple[np.ndarray, int, int]:
    """fold_arrival_order(). states=None folds from None everywhere onto a table of n_agg slots (what fold_unsorted does)."""
    import ctypes as C
    prog = _packed_program(rules, state_bytes, f64_fields)
    recs = np.ascontiguousarray(records).view(np.uint8).reshape(-1)
    if states is None:
        table = np.zeros((int(n_agg), state_bytes), dtype=np.uint8)
    else:
        table = np.ascontiguousarray(states).view(np.uint8).reshape(-1, state_bytes).copy()
    nev, nerr = C.c_uint64(0), C.c_uint64(0)
    rc = _lib().orc_prog_fold_arrival(_ptr(prog), _ptr(recs), recs.size // 64, _ptr(table), table.shape[0], C.addressof(nev), C.addressof(nerr))
    if rc:
        raise ValueError("program oracle: aggregate index out of range" if rc == -1 else "program oracle: out of memory")
    return table, int(nev.value), int(nerr.value)

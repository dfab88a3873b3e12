"""Declarative fold programs (include/sgr.h sgr_fold_program) for the reference's sample models.

Each program is the op-table form of one handleEvent; the docstring quotes the Scala it
stands for. The oracle restates the same handlers directly from the Scala, independently of
these tables — the parity tests check table == handler.
"""
from __future__ import annotations

from typing import Iterable, Sequence, Tuple

from . import native as N


def make_program(state_bytes: int, record_kind: int, rules: Sequence[Tuple[int, Sequence[Tuple[int, int, int, int]]]],
                 f64_fields: Iterable[int] = ()) -> N.sgr_fold_program:
    """rules: [(exists_rule, [(opcode, dst_off, src_off, len), ...]), ...] indexed by event type."""
    p = N.sgr_fold_program()
    p.state_bytes = state_bytes
    p.record_kind = record_kind
    p.n_types = len(rules)
    f64 = list(f64_fields)
    p.n_f64_fields = len(f64)
    for i, off in enumerate(f64):
        p.f64_field_off[i] = off
    for t, (exists_rule, ops) in enumerate(rules):
        r = p.rules[t]
        r.exists_rule = exists_rule
        r.n_ops = len(ops)
        for i, (opcode, dst, src, ln) in enumerate(ops):
            r.ops[i].opcode, r.ops[i].dst_off, r.ops[i].src_off, r.ops[i].len = opcode, dst, src, ln
    return p


def counter_program(record_kind: int = N.REC_FIXED64) -> N.sgr_fold_program:
    """scaladsl TestBoundedContext.scala:77-89
        val current = agg.getOrElse(State(evt.aggregateId, 0, 0))            -> SGR_MATERIALISE
        CountIncremented(_, by, seq) => current.copy(count = count + by, version = seq)
        CountDecremented(_, by, seq) => current.copy(count = count - by, version = seq)
        _: NoOpEvent                 => current
        ExceptionThrowingEvent       => throw e                              -> SGR_THROW
    record: seq @4, by @16; state: count @0, version @4."""
    return make_program(16, record_kind, [
        (N.MATERIALISE, [(N.OP_ADD_I32, 0, 16, 4), (N.OP_SET, 4, 4, 4)]),
        (N.MATERIALISE, [(N.OP_SUB_I32, 0, 16, 4), (N.OP_SET, 4, 4, 4)]),
        (N.MATERIALISE, []),
        (N.THROW, []),
    ])


def ml_counter_program(record_kind: int = N.REC_FIXED64) -> N.sgr_fold_program:
    """multilanguage test TestBoundedContext.scala:68-75: the Counter fold with only the two counting
    event classes; anything else is a scala.MatchError (type >= n_types)."""
    return make_program(16, record_kind, [
        (N.MATERIALISE, [(N.OP_ADD_I32, 0, 16, 4), (N.OP_SET, 4, 4, 4)]),
        (N.MATERIALISE, [(N.OP_SUB_I32, 0, 16, 4), (N.OP_SET, 4, 4, 4)]),
    ])


def bank_account_program() -> N.sgr_fold_program:
    """surge-docs BankAccountCommandModel.scala:81-86
        case create: BankAccountCreated  => Some(BankAccount(number, owner, code, balance))   -> SGR_CREATE
        case updated: BankAccountUpdated => aggregate.map(_.copy(balance = updated.newBalance)) -> SGR_IF_EXISTS
    record: uuid @16, balance @32, owner @40, code @56; state: uuid @0, balance @16, owner @24, code @40.
    balance is a JVM Double: bit-copied, compared with == for the publish rule."""
    return make_program(64, N.REC_FIXED64, [
        (N.CREATE, [(N.OP_SET, 0, 16, 16), (N.OP_SET, 16, 32, 8), (N.OP_SET, 24, 40, 16), (N.OP_SET, 40, 56, 8)]),
        (N.IF_EXISTS, [(N.OP_SET, 16, 32, 8)]),
    ], f64_fields=[16])


def int_balance_program() -> N.sgr_fold_program:
    """multilanguage-scala-sdk-sample Main.scala:25-30
        (None, MoneyDeposited(a))    => Some(BankAccount(a))
        (Some(BankAccount(b)), ...)  => Some(BankAccount(b + a))
    = materialise 0 then add (0 + a == a)."""
    return make_program(16, N.REC_FIXED64, [(N.MATERIALISE, [(N.OP_ADD_I32, 0, 16, 4)])])


def csharp_bank_program() -> N.sgr_fold_program:
    """multilanguage-csharp-sdk Sample/Program.cs:62-80
        var balance = state.IsSome switch { true => state.ToList().Head().amount, _ => 0 };
        return bankEvent switch {
            MoneyWithdrawn m1 => Option<Account>.Some(new Account(balance - m1.Amount)),
            MoneyDeposited m3 => Option<Account>.Some(new Account(balance + m3.Amount)),
            _ => Option<Account>.None
        };
    = materialise 0 then subtract / add (C# int arithmetic wraps, as SUB_I32 / ADD_I32 do). Type 0 MoneyWithdrawn, type 1
    MoneyDeposited, type 2 the `_ => None` arm: a JSON packer maps any other "Type" there with unknown_type = 2.
    record: Amount @16; state: amount @0."""
    return make_program(16, N.REC_FIXED64, [
        (N.MATERIALISE, [(N.OP_SUB_I32, 0, 16, 4)]),
        (N.MATERIALISE, [(N.OP_ADD_I32, 0, 16, 4)]),
        (N.TOMBSTONE, []),
    ])


def counter_snapshot_restore_program() -> N.sgr_fold_program:
    """Today's recovery in the reference: Kafka Streams materialises the compacted STATE topic into a KTable — last
    write wins per key, a null value deletes (modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:57-76;
    null = None state, modules/command-engine/core/src/main/scala/surge/internal/SurgeModel.scala:62-64).
    As a fold over state-snapshot records it is two rules: type 0 (snapshot) = CREATE + SET every state word from the
    record, type 1 (tombstone) = TOMBSTONE. Counter snapshot record: count @16, version @20."""
    return make_program(16, N.REC_FIXED64, [
        (N.CREATE, [(N.OP_SET, 0, 16, 4), (N.OP_SET, 4, 20, 4)]),
        (N.TOMBSTONE, []),
    ])


COUNTER_SNAPSHOT_TYPE, COUNTER_TOMBSTONE_TYPE = 4, 5


def counter_program_with_snapshot_rules() -> N.sgr_fold_program:
    """The Counter handler plus the two rules that let ONE table take both feeds of the state store (shim/scala
    GpuReplayPersistencePlugin.scala): events of the events topic (types 0-3 as in counter_program) and records of the compacted
    STATE topic — type 4 = a snapshot (CREATE + SET every state word from the record: count @16, version @20: last write wins,
    SurgeStateStoreConsumer.scala:57-76), type 5 = a null value (TOMBSTONE: the key is deleted, SurgeModel.scala:62-64)."""
    return make_program(16, N.REC_FIXED64, [
        (N.MATERIALISE, [(N.OP_ADD_I32, 0, 16, 4), (N.OP_SET, 4, 4, 4)]),
        (N.MATERIALISE, [(N.OP_SUB_I32, 0, 16, 4), (N.OP_SET, 4, 4, 4)]),
        (N.MATERIALISE, []),
        (N.THROW, []),
        (N.CREATE, [(N.OP_SET, 0, 16, 4), (N.OP_SET, 4, 20, 4)]),
        (N.TOMBSTONE, []),
    ])

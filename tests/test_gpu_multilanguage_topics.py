"""-m gpu: multilanguage topics whose payloads are the business app's JSON (SGR_VALUE_PROTOBUF_JSON), and state values written in
the same protobuf wrapping (sgr_set_state_writer_framing).

  * events topics of the three reference models (the multilanguage test Counter, the Scala SDK sample, the C# SDK sample):
    about a million records each over four partitions, lz4 and plain batches, an aborted transaction, flush markers and a refetch
    of duplicates. The device decoder must match the host decoder (states, ids, offsets, statistics), and the states must match
    the handlers restated from the apps' sources (oracle/surge_model.py, oracle/multilanguage.py);
  * hostile values on the device give the host's refusal for the batch's first bad record and apply nothing;
  * state topics (the Counter's AggregateState, the C# Account, a 64-byte state with UUID, PSTR and F64 members) restored
    against oracle/multilanguage.read_committed_states;
  * the writer: every value read parses with the protobuf runtime as State(aggregateId = the row's id, payload = the JSON value
    the same read gives unwrapped), capacity counts the wrapper, a row without an id is refused, and a state topic written from
    the wrapped values restores to the same table."""
import json
import re
import struct
import uuid

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import multilanguage as ML
from oracle import state_topic as ST
from oracle import surge_model as SM
from oracle import value_corpus as VC
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200 import synth as SY
from surge_b200.dingest import DeviceIngest
from surge_b200.engine import ReplayEngine
from surge_b200.ingest import Ingest, IngestError
from surge_b200.native import SgrError

pytestmark = pytest.mark.gpu

CH_ERR = N.ST_CHANGED | N.ST_ERROR


def _pb_class(name):
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

    fdp = descriptor_pb2.FileDescriptorProto(name=f"{name}.proto", package="surge.multilanguage", syntax="proto3")
    m = fdp.message_type.add(name=name)
    m.field.add(name="aggregateId", number=1, type=descriptor_pb2.FieldDescriptorProto.TYPE_STRING, label=descriptor_pb2.FieldDescriptorProto.LABEL_OPTIONAL)
    m.field.add(name="payload", number=2, type=descriptor_pb2.FieldDescriptorProto.TYPE_BYTES, label=descriptor_pb2.FieldDescriptorProto.LABEL_OPTIONAL)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName(f"surge.multilanguage.{name}"))


Event, State = _pb_class("Event"), _pb_class("State")


def _wrap(msg, aid, obj):
    return msg(aggregateId=aid, payload=json.dumps(obj, separators=(",", ":")).encode()).SerializeToString()


class _Pair:
    """One device ingest and one host ingest with the same program, packer and framing 3, polled with the same bytes."""

    def __init__(self, prog, packer, unknown_type=-1, max_keys=1 << 17):
        self.dev, self.host = ReplayEngine(0), ReplayEngine(0)
        self.dev.register_program(prog)
        self.host.register_program(prog)
        self.dg, self.ing = DeviceIngest(self.dev, max_keys), Ingest()
        for g in (self.dg, self.ing):
            g.set_json_packer(*packer, unknown_type=unknown_type)
            g.set_value_framing(N.VALUE_PROTOBUF_JSON)
        self.parts = set()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.dg.close()
        self.ing.close()
        self.dev.close()
        self.host.close()

    def poll(self, fetches):
        host_st = {}
        for p, d, aborted in fetches:
            self.dg.set_aborted(p, aborted)
            self.ing.set_aborted(p, aborted)
            self.dg.submit(p, d)
            for k, v in self.ing.record_batches(p, d).items():
                host_st[k] = host_st.get(k, 0) + v
            self.parts.add(p)
        dev_st = self.dg.fold()
        self.host.fold_ingested(self.ing)
        assert {k: v for k, v in dev_st.items() if k != "n_trailing_bytes"} == {k: v for k, v in host_st.items() if k != "n_trailing_bytes"}
        keys = self.ing.keys()
        table, ref = self.dev.export_states(), self.host.export_states()
        _, _, idx = self.dev.get_many(keys, arrays=True)
        assert (idx >= 0).all() and len(set(idx.tolist())) == len(keys)
        assert np.array_equal(table[idx], ref[:len(keys)])
        assert {p: self.dg.offsets(p) for p in self.parts} == {p: self.ing.offsets(p) for p in self.parts}
        return dev_st


# ---------------------------------------------------------------------------------------- 5: events topics at scale
ML_CLS = [c[0] for c in ML.ML_COUNTER_EVENTS[1]]


def _ml_counter_event(rng, agg, seq):
    if rng.random() < 0.6:
        by = int(rng.integers(-2**31, 2**31)) if rng.random() < 0.1 else int(rng.integers(-5, 6))
        return {"_type": ML_CLS[0], "aggregateId": agg, "incrementBy": by, "sequenceNumber": seq}, SM.CountIncremented(agg, by, seq)
    by = int(rng.integers(-5, 6))
    return {"_type": ML_CLS[1], "aggregateId": agg, "decrementBy": by, "sequenceNumber": seq}, SM.CountDecremented(agg, by, seq)


def _int_balance_event(rng, agg, seq):
    a = int(rng.integers(-2**31, 2**31)) if rng.random() < 0.05 else int(rng.integers(-100, 1000))
    return {"amount": a}, SM.MoneyDeposited(a)


def _csharp_event(rng, agg, seq):
    r = rng.random()
    ty = "MoneyDeposited" if r < 0.55 else "MoneyWithdrawn" if r < 0.98 else "MoneyFrozen"
    obj = {"Type": ty, "Amount": int(rng.integers(-50, 500))}
    return obj, ML.csharp_bank_event(obj)


def _ml_state(s):
    return None if s is None else struct.pack("<ii", s.count, s.version)


MODELS = {
    "ml_counter": (P.ml_counter_program, ML.ML_COUNTER_EVENTS, -1, _ml_counter_event, SM.ml_counter_apply_event, _ml_state),
    "int_balance": (P.int_balance_program, ML.INT_BALANCE_EVENTS, -1, _int_balance_event, SM.int_balance_event_handler,
                    lambda s: None if s is None else struct.pack("<i", s.balance) + bytes(4)),
    "csharp_bank": (P.csharp_bank_program, ML.CSHARP_BANK_EVENTS, ML.CSHARP_BANK_UNKNOWN_TYPE, _csharp_event, ML.csharp_bank_event_handler,
                    lambda s: None if s is None else struct.pack("<i", s.amount) + bytes(4)),
}
N_PARTS, DISTINCT, REPEATS, PER_BATCH = 4, 12, 41, 512   # 4 x 12 x 41 x 512 = 1 007 616 records


@pytest.mark.parametrize("name", list(MODELS))
def test_events_topic_device_matches_host_and_the_restated_handler(name):
    prog, packer, unknown, gen, handler, as_row = MODELS[name]
    rng = np.random.default_rng([7, len(name)])
    # per partition: DISTINCT batches of wrapped events (some records are flush markers), reused at rising base offsets; the
    # aggregates of a partition are its own, so its record order is each aggregate's event order
    distinct, objs = {}, {}
    for p in range(N_PARTS):
        for b in range(DISTINCT):
            recs, evs = [], []
            for d in range(PER_BATCH):
                if rng.random() < 0.01:
                    recs.append((d, b"", b""))                      # the producer's flush record
                    continue
                agg = "p%d-%d" % (p, int(rng.integers(0, 3000)))
                obj, ev = gen(rng, agg, int(rng.integers(0, 2**31)))
                recs.append((d, ("%s:%d" % (agg, d)).encode(), _wrap(Event, agg, obj)))
                evs.append((agg, ev))
            distinct[p, b] = K.encode_record_batch(0, recs, compression="lz4" if b % 2 else "none")
            objs[p, b] = evs
    fetches, order, aborted_fetch = [], {p: [] for p in range(N_PARTS)}, None
    for p in range(N_PARTS):
        data, off = bytearray(), 0
        for k in range(DISTINCT * REPEATS):
            b = bytearray(distinct[p, k % DISTINCT])
            b[0:8] = struct.pack(">q", off)
            data += b
            order[p].append(k % DISTINCT)
            off += PER_BATCH
        aborted = []
        if p == 1:   # an aborted transaction with its marker at the end of the fetch
            pid = 77
            data += K.encode_record_batch(off, [(0, b"p1-0", _wrap(Event, "p1-0", gen(rng, "p1-0", 1)[0]))], compression="lz4",
                                          producer_id=pid, producer_epoch=0, transactional=True)
            data += K.encode_control_batch(off + 1, pid, K.ABORT)
            aborted = [(pid, off)]
        fetches.append((p, bytes(data), aborted))
    with _Pair(prog(), packer, unknown) as t:
        half = [(p, d, a) for p, d, a in fetches[:2]]
        st = t.poll(half)
        st2 = t.poll(fetches[2:] + [(0, fetches[0][1], [])])    # partition 0 again: every record a duplicate
        assert st2["n_duplicates"] == DISTINCT * REPEATS * PER_BATCH
        assert st["n_aborted_batches"] == 1 and st["n_markers"] > 0
        total = st["n_records"] + st2["n_records"]
        assert total > 990_000
        # the restated handler, aggregate by aggregate in arrival order
        state = {}
        for p in range(N_PARTS):
            for b in order[p]:
                for agg, ev in objs[p, b]:
                    try:
                        state[agg] = handler(state.get(agg), ev)
                    except ValueError:
                        raise AssertionError("the corpus holds no event the handler throws on")
        keys = sorted(state)
        rows, fl, idx = t.dev.get_many(keys, arrays=True)
        assert (idx >= 0).all()
        for i, k in enumerate(keys):
            want = as_row(state[k])
            if want is None:
                assert not fl[i] & N.ST_EXISTS, k
            else:
                assert fl[i] & N.ST_EXISTS and rows[i, :8].tobytes() == want, (k, state[k], rows[i, :8].tobytes())
        if name == "csharp_bank":
            assert any(state[k] is None for k in keys)              # an unknown Type ends as a tombstone (the `_ => None` arm)


# ------------------------------------------------------------------------------------------ 6: hostile values
def _why(msg):
    return re.sub(r"^[A-Z_]+: (partition -?\d+ )?offset -?\d+(, record \d+)?: ", "", msg)


def test_hostile_values_are_refused_as_the_host_refuses_them_and_apply_nothing():
    rng = np.random.default_rng(66)
    corpus = ML.pbjson_corpus(rng, VC.counter_values(rng), Event)
    core = ("_type", [(n, t, [f[:3] for f in fs]) for n, t, fs in VC.COUNTER])
    with _Pair(P.counter_program(), core, unknown_type=3) as t:
        good = [(b"g%d" % i, _wrap(Event, "g%d" % i, {"_type": VC.T_INC, "incrementBy": i, "sequenceNumber": i})) for i in range(6)]
        t.poll([(0, K.encode_record_batch(0, [(d, k, v) for d, (k, v) in enumerate(good)], compression="lz4"), [])])
        off, refused, whys = 6, 0, set()
        for v in corpus[::7]:
            probe = Ingest()
            try:
                probe.set_json_packer(*core, unknown_type=3)
                probe.set_value_framing(N.VALUE_PROTOBUF_JSON)
                probe.record_batches(0, K.encode_record_batch(0, [(0, b"v", v)]))
                continue                                            # accepted: not a hostile value
            except IngestError:
                pass
            finally:
                probe.close()
            recs = [(d, k, v2) for d, (k, v2) in enumerate(good[:2])] + [(2, b"bad", v), (3, b"bad2", b"\x12\x01x")]
            data = K.encode_record_batch(off, recs, compression="lz4" if refused % 2 else "none")
            with pytest.raises(IngestError) as hi:
                t.ing.record_batches(0, data)
            before, stats = t.dev.export_states(), t.dg.offsets(0)
            with pytest.raises(IngestError) as di:
                t.dg.submit(0, data)
                t.dg.fold()
            assert hi.value.code == di.value.code == N.SGR_ERR_INVALID
            assert re.match(r"^[A-Z_]+: offset %d, record 2: " % off, str(di.value)), str(di.value)
            assert _why(str(hi.value)) == _why(str(di.value)), (str(hi.value), str(di.value))
            assert np.array_equal(t.dev.export_states(), before) and t.dg.offsets(0) == stats == (off, off)
            whys.add(_why(str(di.value)))
            refused += 1
            if refused >= 250:
                break
        assert refused >= 100 and len(whys) >= 8 and "value is not a protobuf Event" in whys
        t.poll([(0, K.encode_record_batch(off, [(d, k, v) for d, (k, v) in enumerate(good)]), [])])   # the next good poll folds


# -------------------------------------------------------------------------------------------- 7: state topics
BIG_STATE = [("id", N.JSON_UUID, 0), ("name", N.JSON_PSTR, 16, 20), ("balance", N.JSON_F64, 40), ("n", N.JSON_I32, 48)]


def _big_obj(rng, aid):
    bal = float(np.frombuffer(rng.bytes(8), "<f8")[0]) if rng.random() < 0.5 else float(rng.choice([0.0, -0.0, 0.1, 1e21, 5e-324]))
    if not np.isfinite(bal):
        bal = 2.5
    name = "".join(rng.choice(list("abZé日😀"), int(rng.integers(0, 5))))
    return {"id": str(uuid.UUID(bytes=rng.bytes(16))), "aggregateId": aid, "name": name, "balance": bal, "n": int(rng.integers(-2**31, 2**31))}


STATE_MODELS = {
    "ml_counter": (16, (), ML.ML_COUNTER_STATE, lambda rng, aid: {"aggregateId": aid, "count": int(rng.integers(-3, 3)), "version": int(rng.integers(0, 3))}),
    "csharp_account": (16, (), ML.CSHARP_ACCOUNT_STATE, lambda rng, aid: {"amount": int(rng.integers(-2, 2))}),
    "big": (64, (40,), BIG_STATE, _big_obj),
}


def _state_program(sb, f64):
    return P.make_program(sb, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 16, 4)]), (N.TOMBSTONE, [])], f64_fields=list(f64))


class _Restore:
    def __init__(self, sb, f64, members):
        self.e = ReplayEngine(0)
        self.e.register_program(_state_program(sb, f64))
        self.sb, self.f64, self.members = sb, f64, members
        self.dg = DeviceIngest(self.e, 1 << 16)
        self.dg.set_state_topic(True)
        self.dg.set_json_packer("", [("State", 0, members)])
        self.dg.set_value_framing(N.VALUE_PROTOBUF_JSON)
        self.fetches, self.n_recs, self.ids, self.table = [], 0, [], np.zeros((0, sb), np.uint8)

    def close(self):
        self.dg.close()
        self.e.close()

    def poll(self, fetches):
        for p, data, aborted in fetches:
            self.dg.set_aborted(p, aborted)
            self.dg.submit(p, data)
        got = self.dg.fold()
        self.fetches += fetches
        recs, nxt, _ = ML.read_committed_states(self.fetches, self.members, self.sb - 8)
        new, self.n_recs = recs[self.n_recs:], len(recs)
        assert got["n_records"] == len(new)
        self.ids, self.table = ST.apply(self.ids, self.table, new, self.f64)
        user = self.sb - 8
        states, fl, idx = self.e.get_many(self.ids, arrays=True)
        assert (idx >= 0).all()
        flags = self.table[:, self.sb - 8:self.sb - 4].copy().view("<u4").ravel()
        assert fl.tolist() == flags.tolist()
        for i in range(len(self.ids)):
            if flags[i] & N.ST_EXISTS:
                a, b = states[i], self.table[i, :user]
                for off in self.f64:                               # doubles by ==
                    assert struct.unpack_from("<d", a, off) == struct.unpack_from("<d", b, off)
                    a, b = a.copy(), b.copy()
                    a[off:off + 8] = 0
                    b[off:off + 8] = 0
                assert a.tobytes() == b.tobytes(), self.ids[i]
        assert {p: self.dg.offsets(p) for p in nxt} == {p: (nxt[p], nxt[p]) for p in nxt}
        return got


def _state_polls(rng, gen, n_polls=4, n_ids=300):
    ids = ["s-%d" % i for i in range(n_ids)] + ["zoë-%d" % i for i in range(20)]
    off, polls = {0: 0, 1: 0}, []
    for _ in range(n_polls):
        poll = []
        for p in (0, 1):
            recs = []
            for d in range(int(rng.integers(200, 700))):
                k = ids[int(rng.integers(0, len(ids)))] if rng.random() < 0.97 else "only-%d" % int(rng.integers(0, 1 << 30))
                if rng.random() < 0.15:
                    recs.append((d, k.encode(), None))               # a tombstone
                else:
                    recs.append((d, k.encode(), _wrap(State, k, gen(rng, k))))   # rewrites of one id inside the poll are common
            poll.append((p, K.encode_record_batch(off[p], recs, compression="lz4" if rng.random() < 0.5 else "none"), []))
            off[p] += len(recs)
        polls.append(poll)
    return polls


@pytest.mark.parametrize("name", list(STATE_MODELS))
def test_state_topic_restore_against_the_restatement(name):
    sb, f64, members, gen = STATE_MODELS[name]
    rng = np.random.default_rng([17, len(name)])
    r = _Restore(sb, f64, members)
    try:
        for poll in _state_polls(rng, gen):
            r.poll(poll)
    finally:
        r.close()


# ---------------------------------------------------------------------------------------------- 8: the writer
def _values_check(e, ids):
    """every value read under both framings: State(aggregateId = id, payload = the JSON read) byte for byte"""
    e.set_state_writer_framing(N.VALUE_JSON)
    js = e.get_many_values(ids)
    ex_js = [(k, v) for pg in e.export_changes_values(CH_ERR, values_cap=1 << 20) for k, v in zip(pg[3], pg[4])]
    sc_js = [(k, v) for pg in e.scan_values(values_cap=1 << 20) for k, v in zip(pg[2], pg[3])]
    e.set_state_writer_framing(N.VALUE_PROTOBUF_JSON)
    pb = e.get_many_values(ids)
    ex_pb = [(k, v) for pg in e.export_changes_values(CH_ERR, values_cap=997) for k, v in zip(pg[3], pg[4])]
    sc_pb = [(k, v) for pg in e.scan_values(values_cap=997) for k, v in zip(pg[2], pg[3])]
    assert len(ex_pb) == len(ex_js) and len(sc_pb) == len(sc_js) and any(v is not None for v in pb)
    for (k, j), (k2, w) in zip(list(zip(ids, js)) + ex_js + sc_js, list(zip(ids, pb)) + ex_pb + sc_pb):
        assert k == k2
        if j is None:
            assert w is None
            continue
        m = State.FromString(w)
        assert m.aggregateId == k and m.payload == j
        assert w == State(aggregateId=k, payload=j).SerializeToString()
    return pb


def test_writer_framing_reads_capacity_refusals_and_round_trip():
    rng = np.random.default_rng(8)
    sb, f64, members, gen = STATE_MODELS["big"]
    r = _Restore(sb, f64, members)
    try:
        for poll in _state_polls(rng, gen, n_polls=2):
            r.poll(poll)
        e = r.e
        with pytest.raises(SgrError) as ei:
            e.set_state_writer_framing(N.VALUE_PROTOBUF_EVENT)
        assert ei.value.code == N.SGR_ERR_INVALID
        e.set_state_writer_framing(N.VALUE_PROTOBUF_JSON)           # before the writer: it survives set_state_writer
        e.set_state_writer([("aggregateId", N.JSON_ID)] + list(members))
        ids = list(r.ids) + ["never-seen"]
        pb = e.get_many_values(ids)
        assert State.FromString(next(v for v in pb if v is not None)).aggregateId
        pb = _values_check(e, ids)
        # capacity and values_len count the wrapper
        need = sum(len(v) for v in pb if v is not None)
        with pytest.raises(SgrError) as ei:
            e.get_many_values(ids, values_cap=need - 1)
        assert ei.value.code == N.SGR_ERR_CAPACITY and str(need) in str(ei.value)
        assert e.get_many_values(ids, values_cap=need) == pb
        # round trip: the wrapped values as an lz4 state topic, restored under framing 3, give the same table
        r2 = _Restore(sb, f64, members)
        try:
            live = [(k, v) for k, v in zip(ids, pb) if v is not None]
            r2.poll([(0, K.encode_record_batch(0, [(d, k.encode(), v) for d, (k, v) in enumerate(live)], compression="lz4"), [])])
            a, fa, _ = e.get_many([k for k, _ in live], arrays=True)
            b, fb, _ = r2.e.get_many([k for k, _ in live], arrays=True)
            for off in f64:   # (-0.0 is written as 0: doubles compare by ==)
                assert [struct.unpack_from("<d", x, off) for x in a] == [struct.unpack_from("<d", x, off) for x in b]
                a[:, off:off + 8] = 0
                b[:, off:off + 8] = 0
            assert np.array_equal(a, b) and (fb & N.ST_EXISTS).all()
        finally:
            r2.close()
        # register_program resets the framing to JSON
        e.register_program(_state_program(sb, f64))
        with pytest.raises(SgrError):
            e.get_many_values(ids)                                  # (and clears the writer)
    finally:
        r.close()
    with ReplayEngine(0) as e:
        with pytest.raises(SgrError) as ei:
            e.set_state_writer_framing(N.VALUE_PROTOBUF_JSON)
        assert ei.value.code == N.SGR_ERR_NO_PROGRAM


def test_rows_without_ids_are_refused_under_the_wrapping():
    counts = np.random.default_rng(2).integers(0, 20, size=3000)
    rec, off = SY.counter_csr(len(counts), counts, seed=9, p_throw=0.0)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_events(rec, off)
        e.fold()
        e.set_state_writer([("count", N.JSON_I32, 0), ("version", N.JSON_I32, 4)])   # no ID member: JSON values need no id
        assert any(v is not None for pg in e.export_changes_values(CH_ERR) for v in pg[4])
        e.set_state_writer_framing(N.VALUE_PROTOBUF_JSON)
        with pytest.raises(SgrError) as ei:
            list(e.export_changes_values(CH_ERR))
        assert ei.value.code == N.SGR_ERR_UNSUPPORTED
        assert "State.aggregateId: the row has no aggregate id in the key table" in str(ei.value), str(ei.value)
        e.load_keys(["agg-%d" % g for g in range(len(counts))])
        vals = [(k, v) for pg in e.export_changes_values(CH_ERR, values_cap=500) for k, v in zip(pg[3], pg[4]) if v is not None]
        assert vals and all(State.FromString(v).aggregateId == k for k, v in vals)

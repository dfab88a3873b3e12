"""-m gpu: which rows carry the CHANGED / ERROR flags of the last operation, over random sequences of operations on one table.

Every operation that writes the table first clears the flags the operation before it left: a fold, set_initial_states or
grow_states leaves the whole table to clear, a sort-based micro-batch or a put batch the rows it touched, an atomic
micro-batch the rows its kernel listed. This pins every pair of consecutive operations to a restatement that clears every
row each time (oracle/program_interp.py for folds, oracle/put_batch.py for put batches and state-topic polls): after each step
the whole table (program bytes, flags, err_idx) and the rows export_changes(CHANGED | ERROR) returns are compared.

The engine refuses some mixes, so each family of operations runs on an engine of its own: put batches number their own ids
(and are refused on a key table that mirrors an ingest's dictionary), a device ingest takes either events or a state topic.
Each family runs a sort-free program (the Counter with its snapshot rules), the same rules on the sort-based path (option
incremental = 1) and a BankAccount-shaped program."""
import struct

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import program_interp as I
from oracle import put_batch as O
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest

pytestmark = pytest.mark.gpu

CH_ERR = N.ST_CHANGED | N.ST_ERROR
N_STEPS = 30

# name -> (program, options, event types the records draw from, a type that throws)
PROGRAMS = {
    "counter": (P.counter_program_with_snapshot_rules, {}, [0, 0, 1, 2, 4, 5], 3),
    "counter_sorted": (P.counter_program_with_snapshot_rules, {"incremental": 1}, [0, 0, 1, 2, 4, 5], 3),
    "bank_account": (P.bank_account_program, {}, [0, 1, 1], 7),
}


def _flags(table):
    return table[:, -8:-4].copy().view("<u4").ravel()


class Run:
    """One engine, its restatement (`table`, None while the engine holds no readable table) and the operations on both."""

    def __init__(self, e, name, rng):
        make, options, self.types, self.throw = PROGRAMS[name]
        prog = make()
        e.register_program(prog)
        for k, v in options.items():
            e.set_option(k, v)
        self.e, self.rng = e, rng
        self.rules = [(prog.rules[t].exists_rule, [(o.opcode, o.dst_off, o.src_off, o.len) for o in prog.rules[t].ops[:prog.rules[t].n_ops]])
                      for t in range(prog.n_types)]
        self.sb, self.f64 = prog.state_bytes, list(prog.f64_field_off[:prog.n_f64_fields])
        self.name, self.table = name, None
        self.known, self.next = {}, 0   # device ingest: the ids polled so far, the next offset

    # ------------------------------------------------------------ inputs
    def records(self, n, n_agg, throws=True):
        """n 64-byte events over aggregates [0, n_agg): type @0, seq @4, aggregate @8, small payload words @16 (Doubles from a
        few values, -0.0 and NaN among them)."""
        rng = self.rng
        r = np.zeros((n, 64), np.uint8)
        for i in range(n):
            t = self.throw if throws and rng.random() < 0.08 else self.types[int(rng.integers(0, len(self.types)))]
            r[i, 16:] = rng.integers(0, 3, size=48, dtype=np.uint8)
            struct.pack_into("<IIQ", r[i], 0, t, i + 1, int(rng.integers(0, n_agg)))
            for off in self.f64:
                struct.pack_into("<d", r[i], off + 16, [0.0, -0.0, 1.5, float("nan")][int(rng.integers(0, 4))])
        return r

    def n_agg(self):
        if self.table is not None and self.rng.random() < 0.6:
            return len(self.table)
        return int(self.rng.integers(1, 80))

    def padded(self, n):
        """The restated table grown to n rows, as the engine grows it: new rows None, no table at all is all None."""
        t = np.zeros((max(n, 0 if self.table is None else len(self.table)), self.sb), np.uint8)
        if self.table is not None:
            t[:len(self.table)] = self.table
        return t

    # ------------------------------------------------------------ every family
    def fold(self):
        n_agg = self.n_agg()
        counts = self.rng.integers(0, 5, size=n_agg)
        recs = self.records(int(counts.sum()), 1)
        offs = np.zeros(n_agg + 1, np.uint64)
        np.cumsum(counts * 64, out=offs[1:])
        self.e.load_events(recs, offs)
        if self.rng.random() < 0.5:
            self.e.fold()
        else:
            self.e.fold_async()
            self.e.wait()
        prior = self.table if self.table is not None and len(self.table) == n_agg else None
        self.table = I.c_fold(self.rules, self.sb, recs, offs, prior, self.f64)[0]

    def set_initial_states(self):
        if self.rng.random() < 0.3:
            self.e.set_initial_states(None)
            self.table = None
            return
        n = int(self.rng.integers(1, 80))
        t = np.zeros((n, self.sb), np.uint8)
        fl = np.array([0, N.ST_EXISTS, N.ST_EXISTS | N.ST_CHANGED, N.ST_EXISTS | N.ST_ERROR], np.uint32)[self.rng.integers(0, 4, size=n)]
        live = (fl & N.ST_EXISTS) != 0
        t[live, :self.sb - 8] = self.rng.integers(0, 3, size=(int(live.sum()), self.sb - 8), dtype=np.uint8)
        t[:, -8:-4] = fl.view(np.uint8).reshape(n, 4)
        t[:, -4:] = (self.rng.integers(0, 3, size=n).astype(np.uint32) * ((fl & N.ST_ERROR) != 0)).view(np.uint8).reshape(n, 4)
        self.e.set_initial_states(t)
        self.table = t

    def grow_states(self):
        have = 0 if self.table is None else len(self.table)
        n = max(1, have + int(self.rng.integers(-3, 40)))
        self.e.grow_states(n)
        if self.table is None or n > len(self.table):
            self.table = self.padded(n)

    def fold_incremental(self):
        if self.table is None:
            with pytest.raises(SgrError) as ex:
                self.e.fold_incremental(self.records(4, 1))
            assert ex.value.code == N.SGR_ERR_NOT_LOADED
            return
        recs = self.records(int(self.rng.integers(1, 40)), len(self.table))
        self.e.fold_incremental(recs)
        self.table = I.c_fold_arrival_order(self.rules, self.sb, recs, self.table, self.f64)[0]

    # ------------------------------------------------------------ engine-numbered ids
    ids = ()

    def put_batch(self):
        rng, user = self.rng, self.sb - 8
        batch = []
        for _ in range(int(rng.integers(1, 30))):
            k = self.ids[int(rng.integers(0, len(self.ids)))] if self.ids and rng.random() < 0.6 else "id-%d" % int(rng.integers(0, 120))
            if rng.random() < 0.25:
                batch.append((k, None))
                continue
            v = bytearray(rng.integers(0, 3, size=user, dtype=np.uint8).tobytes())
            for off in self.f64:
                v[off:off + 8] = struct.pack("<d", [0.0, -0.0, 1.5, float("nan")][int(rng.integers(0, 4))])
            batch.append((k, bytes(v)))
        self.e.put_batch([k for k, _ in batch], [v for _, v in batch], [v is not None for _, v in batch])
        self.ids, self.table, _ = O.put_batch(list(self.ids), self.padded(0), batch, self.f64)

    def fold_unsorted(self):
        n_agg = self.n_agg()
        recs = self.records(int(self.rng.integers(1, 60)), n_agg)
        self.e.set_option("bulk", int(self.rng.integers(0, 2)))
        self.e.fold_unsorted(recs, n_agg)
        self.table = I.c_fold_arrival_order(self.rules, self.sb, recs, None, self.f64, n_agg=n_agg)[0]

    # ------------------------------------------------------------ device ingest
    def poll(self, dg, recs):
        """One poll of (key, value) records through the device ingest, from offset self.next; returns the aggregate index of
        each id in `ids` afterwards."""
        dg.submit(0, K.encode_record_batch(self.next, [(d, k, v) for d, (k, v) in enumerate(recs)],
                                           compression="lz4" if self.rng.random() < 0.5 else "none"))
        self.next += len(recs)
        dg.fold()
        return self.e.get_many(list(self.known), arrays=True)[2]

    def events_poll(self, dg):
        """Events of up to 40 ids (throwing ones among them), with flush markers and null values, which are dropped; one in five
        polls onto a live table has only dropped records."""
        rng = self.rng
        recs, events = [], []
        if self.known and self.table is not None and rng.random() < 0.2:
            recs = [(("%s:0" % next(iter(self.known))).encode(), None), (b"", b"")]
        for d in range(0 if recs else int(rng.integers(1, 30))):
            a = "a%d" % int(rng.integers(0, 40))
            if d and rng.random() < 0.1:
                recs.append((b"", b"") if rng.random() < 0.5 else (("%s:%d" % (a, d)).encode(), None))
                continue
            r = self.records(1, 1)[0]
            recs.append((("%s:%d" % (a, d)).encode(), r[:8].tobytes() + r[16:].tobytes()))
            events.append((a, r))
            self.known.setdefault(a, None)
        idx = dict(zip(self.known, self.poll(dg, recs).tolist()))
        table = self.padded(self.e.n_aggregates())
        if events or self.name == "counter":
            # the sort-free program runs its atomic fold on a poll of dropped records too, which clears the last flags; a grouped
            # program folds nothing there
            live = np.array([r for _, r in events], np.uint8).reshape(-1, 64)
            for i, (a, _) in enumerate(events):
                struct.pack_into("<Q", live[i], 8, idx[a])
            table = I.c_fold_arrival_order(self.rules, self.sb, live, table, self.f64)[0]
        self.table = table

    def state_poll(self, dg):
        """State records of up to 40 ids, tombstones among them; one in five polls onto a live table holds only a flush marker."""
        rng, user = self.rng, self.sb - 8
        recs, batch = [], []
        if self.known and self.table is not None and rng.random() < 0.2:
            recs.append((b"", b""))
        else:
            for _ in range(int(rng.integers(1, 30))):
                k = "s%d" % int(rng.integers(0, 40))
                v = None
                if rng.random() > 0.25:
                    b = bytearray(rng.integers(0, 3, size=user, dtype=np.uint8).tobytes())
                    for off in self.f64:
                        b[off:off + 8] = struct.pack("<d", [0.0, -0.0, 1.5, float("nan")][int(rng.integers(0, 4))])
                    v = bytes(b)
                recs.append((k.encode(), v))
                batch.append((k, v))
                self.known.setdefault(k, None)
        idx = self.poll(dg, recs).tolist()
        table = self.padded(self.e.n_aggregates())
        if batch:
            ids = [None] * len(idx)
            for k, i in zip(self.known, idx):
                ids[i] = k
            table = O.put_batch(ids, table, batch, self.f64)[1]
        self.table = table

    # ------------------------------------------------------------ the check after each step
    def check(self):
        e = self.e
        if self.table is None:
            with pytest.raises(SgrError) as ex:
                e.export_states()
            assert ex.value.code == N.SGR_ERR_STATE
            return
        got = e.export_states()
        assert got.shape == self.table.shape
        bad = np.nonzero((got != self.table).any(axis=1))[0]
        assert not len(bad), f"rows {bad[:8].tolist()}: engine {got[bad[:2]].tolist()} restatement {self.table[bad[:2]].tolist()}"
        flagged = [int(i) for page in e.export_changes(CH_ERR, page_rows=None) for i in page[0]]
        assert flagged == np.nonzero(_flags(self.table) & CH_ERR)[0].tolist()


def _drive(family, name, seed):
    rng = np.random.default_rng(seed)
    with ReplayEngine(0) as e:
        run = Run(e, name, rng)
        common = [run.fold, run.fold, run.set_initial_states, run.grow_states, run.fold_incremental, run.fold_incremental]
        dg = None
        if family == "ids":
            ops = common + [run.put_batch, run.put_batch, run.put_batch, run.fold_unsorted, run.fold_unsorted]
        else:
            dg = DeviceIngest(e, 1 << 12)
            if family == "state_topic":
                dg.set_state_topic(True)
            poll = run.events_poll if family == "events" else run.state_poll
            ops = common + [lambda: poll(dg)] * 4
        try:
            done = []
            for step in range(N_STEPS):
                op = ops[int(rng.integers(0, len(ops)))]
                done.append(getattr(op, "__name__", "poll"))
                op()
                try:
                    run.check()
                except AssertionError as err:
                    raise AssertionError(f"after {done}: {err}") from None
        finally:
            if dg is not None:
                dg.close()


@pytest.mark.parametrize("name", list(PROGRAMS))
@pytest.mark.parametrize("family", ["ids", "events", "state_topic"])
@pytest.mark.parametrize("seed", [1, 2])
def test_each_operation_clears_the_flags_of_the_one_before(family, name, seed):
    _drive(family, name, seed)

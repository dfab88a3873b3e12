"""-m gpu: random fold programs against the program interpreter (oracle/program_interp.py), every kernel.

The sample models only exercise a handful of rule/op combinations. Here the program itself is drawn at random — state
width, exists-rules, SET/ADD/SUB ops (32- and 64-bit), overlapping destinations, Double fields — and the same log is
folded by whichever kernel the engine picks (fold_runs.cu inside the transformer algebra, fold_kernels.cu outside),
by the forced lane-sequential kernel, by the rows kernel, with and without prior states, as an arrival-order load, and
as micro-batches; every state table must equal the interpreter's byte for byte.
"""
import numpy as np
import pytest

from oracle import program_interp as I
from oracle.program_corpus import draw_log, draw_program, draw_var_log, draw_var_program, interleave
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P

pytestmark = pytest.mark.gpu


def same(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(want)} states differ; first {bad[:6]}\n got {got[bad[0]].tolist()}\nwant {want[bad[0]].tolist()}")


@pytest.mark.parametrize("seed", range(40))
def test_random_program_all_paths(seed):
    rng = np.random.default_rng(9000 + seed)
    state_bytes, rules, f64 = draw_program(rng)
    prog = P.make_program(state_bytes, N.REC_FIXED64, rules, f64_fields=f64)
    n_agg = 260
    rec, off, aggs = draw_log(rng, len(rules), n_agg, 700, f64)
    want = I.fold(rules, state_bytes, rec, off, f64_fields=f64)
    what = f"seed {seed} state_bytes {state_bytes} rules {rules} f64 {f64}"
    with ReplayEngine(0) as e:
        e.register_program(prog)
        taken = []
        for kernel in (0, 1, 2, 3):
            e.set_option("kernel", kernel)
            e.set_initial_states(None)
            e.load_events(rec, off)
            try:
                e.fold()
            except SgrError as err:      # a FORCED record-parallel kernel declines programs outside its algebra; auto never does
                assert kernel in (2, 3) and err.code == N.SGR_ERR_UNSUPPORTED, f"{what} kernel {kernel}: {err}"
                continue
            taken.append(kernel)
            same(e.export_states(), want, f"{what} kernel {kernel}")
        assert 0 in taken and 1 in taken
        # a second log on top of the first table (prior states, publish rule against them)
        rec2, off2, _ = draw_log(rng, len(rules), n_agg, 300, f64)
        want2 = I.fold(rules, state_bytes, rec2, off2, initial=want, f64_fields=f64)
        for kernel in [k for k in taken if k != 3]:
            e.set_option("kernel", kernel)
            e.set_initial_states(want)
            e.load_events(rec2, off2)
            e.fold()
            same(e.export_states(), want2, f"{what} kernel {kernel} with prior states")
        e.set_option("kernel", 0)
        # the same first log in arrival order: interleave the aggregates, keep each one's own order
        perm = interleave(rng, aggs)
        e.set_initial_states(None)
        e.fold_unsorted(rec[perm], n_agg)
        same(e.export_states(), want, f"{what} fold_unsorted")
        # micro-batches onto the live table
        table = want
        for b in range(3):
            recb, _, aggb = draw_log(rng, len(rules), n_agg, [40, 400, 5][b], f64)
            pb = interleave(rng, aggb)
            batch = recb[pb]
            table = I.fold_arrival_order(rules, state_bytes, batch, table, f64_fields=f64)
            e.fold_incremental(batch)
            same(e.export_states(), table, f"{what} micro-batch {b}")


# ------------------------------------------------------------------ variable records (SGR_REC_VAR16)
@pytest.mark.parametrize("seed", range(16))
def test_random_program_variable_records(seed):
    rng = np.random.default_rng(7000 + seed)
    state_bytes, rules = draw_var_program(rng)
    prog = P.make_program(state_bytes, N.REC_VAR16, rules)
    n_agg = 300
    buf, seg, rec_off = draw_var_log(rng, len(rules), n_agg, 900)
    want = I.fold_var(rules, state_bytes, buf, seg)
    what = f"seed {seed} state_bytes {state_bytes} rules {rules}"
    with ReplayEngine(0) as e:
        e.register_program(prog)
        for kernel in (0, 1):
            e.set_option("kernel", kernel)
            e.set_initial_states(None)
            e.load_events(buf, seg)
            e.fold()
            same(e.export_states(), want, f"{what} kernel {kernel}")
        e.set_option("kernel", 0)
        e.set_initial_states(None)
        e.load_events_indexed(buf, seg, rec_off)       # with the record directory: the record-parallel kernel where it applies
        e.fold()
        same(e.export_states(), want, f"{what} with directory")
        buf2, seg2, rec_off2 = draw_var_log(rng, len(rules), n_agg, 200)
        want2 = I.fold_var(rules, state_bytes, buf2, seg2, initial=want)
        e.set_initial_states(want)
        e.load_events_indexed(buf2, seg2, rec_off2)
        e.fold()
        same(e.export_states(), want2, f"{what} with prior states")

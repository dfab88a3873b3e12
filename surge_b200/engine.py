"""ReplayEngine: one sgr_engine handle behind a small Python surface.

Host arrays (numpy) go through the host-buffer entry points (H2D/D2H inside the call, what a
JNI caller with direct ByteBuffers would use); CUDA tensors go through the `_device`
entry points and are borrowed, not copied.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import native as N


def _is_cuda_tensor(x) -> bool:
    return hasattr(x, "is_cuda") and bool(getattr(x, "is_cuda"))


def _borrow(t) -> Tuple[object, int]:
    """A CUDA tensor argument as the `_device` entry points borrow it: flat and contiguous, with its byte count. The engine
    launches on its own non-blocking stream and those entry points take plain pointers, which cannot order against torch's
    stream: so what torch is still writing on ITS current stream is waited for first."""
    import torch

    flat = t.contiguous().view(-1)
    if _is_cuda_tensor(flat):
        torch.cuda.current_stream(flat.device).synchronize()
    return flat, flat.numel() * flat.element_size()


def _host_bytes(a) -> np.ndarray:
    return np.ascontiguousarray(a).view(np.uint8).reshape(-1)


def _id_batch(enc: Sequence[bytes]) -> Tuple[np.ndarray, np.ndarray]:
    """A batch of encoded ids as the C ABI takes it: (blob u8, offsets u32[n + 1]), id i = blob[offsets[i]:offsets[i + 1]].
    The blob views the joined bytes without copying them (the C side only reads it) and is never empty, so its pointer is
    never NULL."""
    offs = np.zeros(len(enc) + 1, dtype=np.uint32)
    np.cumsum([len(b) for b in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8), offs


def _rows_or_none(states: np.ndarray, flags: np.ndarray) -> List[Optional[bytes]]:
    """Rows of a batched read as getAggregateBytes answers: the program bytes, or None when the state does not exist."""
    return [states[i].tobytes() if flags[i] & N.ST_EXISTS else None for i in range(len(flags))]


def _split_values(buf: np.ndarray, offs: np.ndarray, n: int) -> List[Optional[bytes]]:
    raw = buf[:int(offs[n])].tobytes() if n else b""
    return [raw[offs[i]:offs[i + 1]] if offs[i + 1] > offs[i] else None for i in range(n)]


class _Page:
    """The buffers one page of an export or a scan is written into. Its rows are the program bytes, or with values_cap the JSON
    values of the *_values twin, whose arguments in their place (values, values_cap, value_offsets) `out` holds."""

    def __init__(self, cap: int, user: int, ids_cap: int, values_cap: Optional[int]):
        if values_cap is None:
            self.rows, self.voffs = np.empty((cap, user), dtype=np.uint8), None
            self.out = (self.rows.ctypes.data,)
        else:
            self.rows, self.voffs = np.empty(max(values_cap, 1), dtype=np.uint8), np.empty(cap + 1, dtype=np.uint64)
            self.out = (self.rows.ctypes.data, values_cap, self.voffs.ctypes.data)
        self.flags = np.empty(cap, dtype=np.uint32)
        self.idx = np.empty(cap, dtype=np.int64)
        self.offs = np.empty(cap + 1, dtype=np.uint32)
        self.blob = np.empty(max(ids_cap, 1), dtype=np.uint8)

    def data(self, k: int):
        return self.rows[:k] if self.voffs is None else _split_values(self.rows, self.voffs, k)

    def ids(self, k: int, n_keys: Optional[int] = None) -> List[Optional[str]]:
        """The page's ids; with n_keys, None for a row at or past the key table (its empty span is told apart from the id "" by its
        index)."""
        offs = self.offs
        raw = self.blob[:int(offs[k])].tobytes() if k else b""
        if n_keys is None:
            return [raw[offs[i]:offs[i + 1]].decode("utf-8") for i in range(k)]
        return [raw[offs[i]:offs[i + 1]].decode("utf-8") if self.idx[i] < n_keys else None for i in range(k)]


class _DevView:
    """Exposes a raw device pointer through __cuda_array_interface__ (for torch.as_tensor)."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}
        self._owner = owner


class ReplayEngine:
    def __init__(self, device: int = 0):
        self._lib = N.load_library()
        self._h = C.c_void_p()
        cfg = N.sgr_config()
        cfg.device = device
        rc = self._lib.sgr_create(C.byref(cfg), C.byref(self._h))
        if rc != N.SGR_OK:
            self._h = C.c_void_p()
            N.check(self._lib, None, rc)
        self.device = device
        self.state_bytes = 0
        self._keep = []  # borrowed device tensors kept alive

    # -- lifecycle
    def close(self) -> None:
        if self._h:
            self._lib.sgr_destroy(self._h)
            self._h = C.c_void_p()
            self._keep = []

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc: int) -> None:
        N.check(self._lib, self._h, rc)

    def _lend(self, t, *also) -> Tuple[int, int]:
        """Borrow a CUDA tensor for a load or a rebuild: the engine may read it until the next one, so it and `also` replace
        the kept tensors. Returns (pointer, bytes)."""
        flat, nbytes = _borrow(t)
        self._keep = [flat, *also]
        return flat.data_ptr(), nbytes

    # -- program
    def register_program(self, prog: N.sgr_fold_program) -> None:
        self._ck(self._lib.sgr_register_program(self._h, C.byref(prog)))
        self.state_bytes = int(prog.state_bytes)

    # -- loads
    def load_events(self, events, seg_offsets) -> None:
        """CSR event log. numpy -> copied to HBM; CUDA tensors -> borrowed, and must not be modified while loaded: the engine
        may fold from a copy of the record words its program reads (include/sgr.h, planes). Load again to fold changed
        records."""
        if _is_cuda_tensor(events):
            assert _is_cuda_tensor(seg_offsets)
            ev, nbytes = self._lend(events, seg_offsets)
            self._ck(self._lib.sgr_load_events_device(self._h, ev, nbytes, seg_offsets.data_ptr(), seg_offsets.numel() - 1))
            return
        ev = _host_bytes(events)
        off = np.ascontiguousarray(seg_offsets, dtype=np.uint64)
        self._ck(self._lib.sgr_load_events(self._h, ev.ctypes.data, ev.size, off.ctypes.data, len(off) - 1))

    def load_events_indexed(self, events, seg_offsets, rec_offsets) -> None:
        """Variable records + record directory (rec_offsets[n_records+1]): enables the record-parallel kernel."""
        if _is_cuda_tensor(events):
            ev, nbytes = self._lend(events, seg_offsets, rec_offsets)
            self._ck(self._lib.sgr_load_events_indexed_device(self._h, ev, nbytes, seg_offsets.data_ptr(), seg_offsets.numel() - 1,
                                                              rec_offsets.data_ptr(), rec_offsets.numel() - 1))
            return
        ev = _host_bytes(events)
        off = np.ascontiguousarray(seg_offsets, dtype=np.uint64)
        ro = np.ascontiguousarray(rec_offsets, dtype=np.uint64)
        self._ck(self._lib.sgr_load_events_indexed(self._h, ev.ctypes.data, ev.size, off.ctypes.data, len(off) - 1, ro.ctypes.data, len(ro) - 1))

    def load_unsorted(self, records, n_agg: int) -> None:
        """Fixed 64-byte records in arrival order; grouped stably by aggregate on the device."""
        if _is_cuda_tensor(records):
            r, nbytes = self._lend(records)
            self._ck(self._lib.sgr_load_unsorted_device(self._h, r, nbytes // 64, n_agg))
            return
        r = _host_bytes(records)
        self._ck(self._lib.sgr_load_unsorted(self._h, r.ctypes.data, r.size // 64, n_agg))

    def fold_unsorted(self, records, n_agg: int) -> None:
        """Rebuild all states from an arrival-order log (Kafka partition order) in one call."""
        if _is_cuda_tensor(records):
            r, nbytes = self._lend(records)
            self._ck(self._lib.sgr_fold_unsorted_device(self._h, r, nbytes // 64, n_agg))
            return
        r = _host_bytes(records)
        self._ck(self._lib.sgr_fold_unsorted(self._h, r.ctypes.data, r.size // 64, n_agg))

    def set_initial_states(self, states: Optional[np.ndarray]) -> None:
        if states is None:
            self._ck(self._lib.sgr_set_initial_states(self._h, None, 0))
            return
        s = np.ascontiguousarray(states).view(np.uint8).reshape(-1, self.state_bytes)
        self._ck(self._lib.sgr_set_initial_states(self._h, s.ctypes.data, s.shape[0]))

    # -- compute
    def fold(self) -> None:
        self._ck(self._lib.sgr_fold(self._h))

    def fold_async(self) -> None:
        """Enqueue the fold on the engine's stream without waiting (pair with wait())."""
        self._ck(self._lib.sgr_fold_async(self._h))

    def wait(self) -> None:
        self._ck(self._lib.sgr_wait(self._h))

    def fold_incremental(self, records) -> None:
        if _is_cuda_tensor(records):
            # the micro-batch is read only during the call; the loaded log's tensors stay kept
            r, nbytes = _borrow(records)
            self._keep.append(r)
            self._ck(self._lib.sgr_fold_incremental_device(self._h, r.data_ptr(), nbytes // 64))
            self._keep.pop()
            return
        r = _host_bytes(records)
        self._ck(self._lib.sgr_fold_incremental(self._h, r.ctypes.data, r.size // 64))

    def grow_states(self, n_agg: int) -> None:
        """Resize the live table on the device, keeping its content (new slots are None)."""
        self._ck(self._lib.sgr_grow_states(self._h, n_agg))

    def fold_ingested(self, ingest) -> None:
        """Fold everything pending in an Ingest onto the live table and publish its id dictionary to get()."""
        self._ck(self._lib.sgr_fold_ingested(self._h, ingest.handle))

    # -- results
    def _states_device(self) -> Tuple[int, int, int]:
        """(device pointer, n_agg, state_bytes) of the live state table."""
        p, n, sb = C.c_void_p(), C.c_uint64(), C.c_uint32()
        self._ck(self._lib.sgr_states_device(self._h, C.byref(p), C.byref(n), C.byref(sb)))
        return p.value, int(n.value), int(sb.value)

    def n_aggregates(self) -> int:
        return self._states_device()[1]

    def export_states(self, out: Optional[np.ndarray] = None, bitmaps: bool = False):
        n = self.n_aggregates()
        if out is None:
            out = np.empty((n, self.state_bytes), dtype=np.uint8)
        if not bitmaps:
            self._ck(self._lib.sgr_export_states(self._h, out.ctypes.data, out.nbytes, None, None, None))
            return out
        nb = (n + 7) // 8
        ex, ch, er = (np.zeros(nb, dtype=np.uint8) for _ in range(3))
        self._ck(self._lib.sgr_export_states(self._h, out.ctypes.data, out.nbytes, ex.ctypes.data, ch.ctypes.data, er.ctypes.data))
        return out, ex, ch, er

    def states_tensor(self):
        """The live device state table as a torch uint8 tensor [n_agg, state_bytes] (borrowed)."""
        import torch

        p, n, sb = self._states_device()
        return torch.as_tensor(_DevView(p, n * sb, self), device=f"cuda:{self.device}").view(n, sb)

    def events_tensors(self):
        """(events u8[nbytes], seg_offsets i64[n_agg+1]) device tensors of the engine's CSR log (borrowed)."""
        import torch

        p, nb, po = C.c_void_p(), C.c_uint64(), C.c_void_p()
        self._ck(self._lib.sgr_events_device(self._h, C.byref(p), C.byref(nb), C.byref(po)))
        ev = torch.as_tensor(_DevView(p.value, nb.value, self), device=f"cuda:{self.device}")
        return ev, po.value

    def load_keys(self, keys: Sequence[str]) -> None:
        blob, offs = _id_batch([k.encode("utf-8") for k in keys])
        self._ck(self._lib.sgr_load_keys(self._h, blob.ctypes.data, offs.ctypes.data, len(offs) - 1))

    def get(self, key: str) -> Optional[bytes]:
        """getAggregateBytes(aggregateId): Option[Array[Byte]] — None when the state does not exist."""
        kb = key.encode("utf-8")
        buf = C.create_string_buffer(N.MAX_STATE_BYTES)
        outlen, exists = C.c_uint32(), C.c_int32()
        kbuf = C.create_string_buffer(kb, len(kb)) if kb else None
        self._ck(self._lib.sgr_get(self._h, C.cast(kbuf, C.c_void_p) if kbuf else None, len(kb), buf, N.MAX_STATE_BYTES,
                                   C.byref(outlen), C.byref(exists)))
        return bytes(buf.raw[:outlen.value]) if exists.value else None

    def get_many(self, keys: Sequence[str], arrays: bool = False):
        """getAggregateBytes for many ids in one call, served from the device table (sgr_get_batch): a list of Optional[bytes],
        the same as get() for each id. arrays=True: (states u8[n, state_bytes - 8], flags u32[n], indices i64[n]) instead, with
        zero rows for None states and unknown ids, flags 0 and index -1 for unknown ids."""
        blob, offs = _id_batch([k.encode("utf-8") for k in keys])
        n = len(offs) - 1
        states = np.zeros((n, max(self.state_bytes - 8, 0)), dtype=np.uint8)
        flags = np.zeros(n, dtype=np.uint32)
        indices = np.zeros(n, dtype=np.int64)
        self._ck(self._lib.sgr_get_batch(self._h, blob.ctypes.data, offs.ctypes.data, n, states.ctypes.data, states.nbytes,
                                         flags.ctypes.data, indices.ctypes.data))
        return (states, flags, indices) if arrays else _rows_or_none(states, flags)

    def put_batch(self, ids: Sequence[str], rows, present=None) -> int:
        """Records of a state topic, in arrival order, applied to the table on the device (sgr_put_batch): the last write per id
        wins, a tombstone (present[i] false) leaves None. rows: u8[n, state_bytes - 8] (or n rows of bytes) holding the program
        bytes; present: bool[n], None for all rows present. New ids get the next dense indices in order of first appearance and
        join the key table get() / get_many() / export_changes() / scan() read. Returns the number of new ids."""
        blob, offs = _id_batch([k.encode("utf-8") for k in ids])
        n = len(offs) - 1
        user = self.state_bytes - 8
        if isinstance(rows, np.ndarray):
            r = np.ascontiguousarray(rows, dtype=np.uint8).reshape(n, user)
        else:
            r = np.zeros((n, user), dtype=np.uint8)
            for i, b in enumerate(rows):
                if b is not None:
                    r[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
        p = np.ones(n, dtype=np.uint8) if present is None else np.ascontiguousarray(present, dtype=bool).astype(np.uint8)
        if r.size == 0:
            r = np.zeros(1, dtype=np.uint8)
        n_new = C.c_uint64()
        self._ck(self._lib.sgr_put_batch(self._h, blob.ctypes.data, offs.ctypes.data, n, r.ctypes.data, p.ctypes.data, C.byref(n_new)))
        return int(n_new.value)

    def export_changes(self, select: int = N.ST_CHANGED, page_rows: Optional[int] = 1 << 20,
                       page_id_bytes: int = 64 << 20) -> Iterator[Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, List[Optional[str]]]]:
        """The aggregates the last fold changed (select=ST_CHANGED) or failed (ST_ERROR, or both), compacted on the device
        (sgr_export_changes). Yields pages of (indices i64[n], flags u32[n], err_idx u32[n], rows u8[n, state_bytes - 8], ids) in
        ascending dense index; ids[i] is the aggregate id (str), or None for a row past the key table. A row is all zero when its
        state is None. A page holds at most page_rows rows (None: the whole table) and page_id_bytes id bytes. Every page of one
        export reads the same table: a fold, grow, set_initial_states or load_keys between two pages raises
        InvalidStateStoreException (SGR_ERR_STATE) from the next one."""
        for idx, flags, err, ids, rows in self._export_pages(select, page_rows, page_id_bytes):
            yield idx, flags, err, rows, ids

    def _export_pages(self, select: int, max_rows: Optional[int], ids_cap: int, values_cap: Optional[int] = None):
        """The pages of sgr_export_changes, or with values_cap of sgr_export_changes_values: (indices, flags, err_idx, ids, rows
        or values). The export ends when the cursor reaches the end of the table."""
        n_agg = self.n_aggregates()
        cap = max(1, n_agg if max_rows is None else min(int(max_rows), max(n_agg, 1)))
        ids_cap = int(ids_cap)
        values_cap = None if values_cap is None else int(values_cap)
        fn = self._lib.sgr_export_changes if values_cap is None else self._lib.sgr_export_changes_values
        cur = N.sgr_changes_cursor()
        n = C.c_uint64()
        while True:
            pg = _Page(cap, self.state_bytes - 8, ids_cap, values_cap)
            err = np.empty(cap, dtype=np.uint32)
            self._ck(fn(self._h, int(select), C.byref(cur), cap, *pg.out, pg.flags.ctypes.data, err.ctypes.data, pg.idx.ctypes.data,
                        pg.blob.ctypes.data, ids_cap, pg.offs.ctypes.data, C.byref(n)))
            k = int(n.value)
            ids = pg.ids(k, int(cur.n_keys))
            if k:
                yield pg.idx[:k], pg.flags[:k], err[:k], ids, pg.data(k)
            if cur.next >= n_agg:
                return

    def scan(self, frm: Optional[str] = None, to: Optional[str] = None, page_rows: int = 1 << 20,
             page_id_bytes: int = 64 << 20) -> Iterator[Tuple[np.ndarray, np.ndarray, np.ndarray, List[str]]]:
        """The live aggregates (their state exists) whose id lies in [frm, to], in Bytes order of the ids (sgr_scan); None leaves
        that end open. Yields pages of (indices i64[n], flags u32[n], rows u8[n, state_bytes - 8], ids), at most page_rows rows
        and page_id_bytes id bytes each. Each page resumes after the last id of the one before, so folds between pages are
        fine: an id live throughout is reported exactly once."""
        for idx, flags, ids, rows in self._scan_pages(frm, to, page_rows, page_id_bytes):
            yield idx, flags, rows, ids

    def _scan_pages(self, frm: Optional[str], to: Optional[str], max_rows: int, ids_cap: int, values_cap: Optional[int] = None):
        """The pages of sgr_scan, or with values_cap of sgr_scan_values: (indices, flags, ids, rows or values). Each page resumes
        after the last id of the one before (from_exclusive); the scan ends on a page that left no live row in range out."""
        n_agg = self.n_aggregates()
        cap = max(1, min(int(max_rows), max(n_agg, 1)))
        ids_cap = int(ids_cap)
        values_cap = None if values_cap is None else int(values_cap)
        fn = self._lib.sgr_scan if values_cap is None else self._lib.sgr_scan_values
        lo = None if frm is None else frm.encode("utf-8")
        hi = None if to is None else to.encode("utf-8")
        hi_buf = None if hi is None else C.create_string_buffer(hi, max(len(hi), 1))
        exclusive = 0
        n, more = C.c_uint64(), C.c_int32()
        while True:
            pg = _Page(cap, self.state_bytes - 8, ids_cap, values_cap)
            lo_buf = None if lo is None else C.create_string_buffer(lo, max(len(lo), 1))
            self._ck(fn(self._h, lo_buf, 0 if lo is None else len(lo), exclusive, hi_buf, 0 if hi is None else len(hi), cap, *pg.out,
                        pg.flags.ctypes.data, pg.idx.ctypes.data, pg.blob.ctypes.data, ids_cap, pg.offs.ctypes.data, C.byref(n), C.byref(more)))
            k = int(n.value)
            if k:
                yield pg.idx[:k], pg.flags[:k], pg.ids(k), pg.data(k)
                lo, exclusive = pg.blob[int(pg.offs[k - 1]):int(pg.offs[k])].tobytes(), 1
            if not more.value:
                return

    # -- JSON state values (sgr_set_state_writer)
    def set_state_writer(self, members) -> None:
        """Register the table the value-returning reads write rows with: members in value order, each (name, N.JSON_*, program
        byte offset[, slot bytes for JSON_PSTR]) or (name, N.JSON_ID) for the aggregate id. An empty table clears the writer."""
        arr = (N.sgr_json_field * max(len(members), 1))()
        names = [m[0].encode("utf-8") for m in members]
        for i, m in enumerate(members):
            arr[i].name = names[i]
            arr[i].kind = m[1]
            if m[1] != N.JSON_ID:
                arr[i].dst_off = m[2]
                arr[i].len = m[3] if len(m) > 3 else 0
        self._ck(self._lib.sgr_set_state_writer(self._h, arr, len(members)))

    def set_state_writer_framing(self, framing: int) -> None:
        """How the value-returning reads wrap the JSON value: N.VALUE_JSON (the default) returns it as it is;
        N.VALUE_PROTOBUF_JSON returns the multilanguage protobuf State{aggregateId = the row's id, payload = the JSON value}, what a
        multilanguage store hands the gateway and republishes. The setting survives set_state_writer; register_program resets it
        to N.VALUE_JSON."""
        self._ck(self._lib.sgr_set_state_writer_framing(self._h, framing))

    def get_many_values(self, keys: Sequence[str], values_cap: Optional[int] = None) -> List[Optional[bytes]]:
        """The JSON state value of each id (sgr_get_batch_values), None for a None state or an unknown id. values_cap: the byte
        budget of one call (None: sized from the first attempt)."""
        blob, offs = _id_batch([k.encode("utf-8") for k in keys])
        n = len(offs) - 1
        flags = np.zeros(max(n, 1), dtype=np.uint32)
        voffs = np.zeros(n + 1, dtype=np.uint64)
        need = C.c_uint64()
        cap = int(values_cap) if values_cap is not None else 64 * n + 64
        while True:
            buf = np.empty(max(cap, 1), dtype=np.uint8)
            rc = self._lib.sgr_get_batch_values(self._h, blob.ctypes.data, offs.ctypes.data, n, buf.ctypes.data, cap, voffs.ctypes.data,
                                                flags.ctypes.data, None, C.byref(need))
            if rc == N.SGR_ERR_CAPACITY and values_cap is None:
                cap = int(need.value)
                continue
            self._ck(rc)
            return _split_values(buf, voffs, n)

    def export_changes_values(self, select: int = N.ST_CHANGED, max_rows: Optional[int] = 1 << 20, values_cap: int = 64 << 20,
                              page_id_bytes: int = 64 << 20) -> Iterator[Tuple[np.ndarray, np.ndarray, np.ndarray, List[Optional[str]], List[Optional[bytes]]]]:
        """export_changes with JSON values in place of rows (sgr_export_changes_values). Yields pages of (indices i64[n], flags
        u32[n], err_idx u32[n], ids, values): values[i] is the row's JSON state, or None for a None state (the tombstone: the
        (id, null) record of a republish). A page also ends before a value that does not fit in values_cap bytes."""
        yield from self._export_pages(select, max_rows, page_id_bytes, values_cap)

    def scan_values(self, frm: Optional[str] = None, to: Optional[str] = None, max_rows: int = 1 << 20, values_cap: int = 64 << 20,
                    page_id_bytes: int = 64 << 20) -> Iterator[Tuple[np.ndarray, np.ndarray, List[str], List[bytes]]]:
        """scan with JSON values in place of rows (sgr_scan_values). Yields pages of (indices i64[n], flags u32[n], ids, values)."""
        yield from self._scan_pages(frm, to, max_rows, page_id_bytes, values_cap)

    def get_index(self, agg: int) -> Tuple[Optional[bytes], int, int]:
        """(program bytes or None, flags, err_idx) of one dense aggregate index."""
        buf = C.create_string_buffer(N.MAX_STATE_BYTES)
        outlen, exists, flags, err = C.c_uint32(), C.c_int32(), C.c_uint32(), C.c_uint32()
        self._ck(self._lib.sgr_get_index(self._h, agg, buf, N.MAX_STATE_BYTES, C.byref(outlen), C.byref(exists),
                                         C.byref(flags), C.byref(err)))
        return (bytes(buf.raw[:outlen.value]) if exists.value else None), int(flags.value), int(err.value)

    # -- multi-GPU (one process per GPU)
    def dist_init(self, rank: int, nranks: int, unique_id: Optional[bytes], recv_capacity_records: int) -> None:
        buf = C.create_string_buffer(unique_id, 128) if unique_id else None
        self._ck(self._lib.sgr_dist_init(self._h, rank, nranks, buf, recv_capacity_records))

    def dist_set_partitions(self, partition_of_agg: np.ndarray) -> None:
        p = np.ascontiguousarray(partition_of_agg, dtype=np.uint32)
        self._ck(self._lib.sgr_dist_set_partitions(self._h, p.ctypes.data, len(p)))

    def dist_ipc_export(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._ck(self._lib.sgr_dist_ipc_export(self._h, buf))
        return bytes(buf.raw)

    def dist_ipc_import(self, handles: Sequence[bytes]) -> None:
        blob = C.create_string_buffer(b"".join(handles), 64 * len(handles))
        self._ck(self._lib.sgr_dist_ipc_import(self._h, blob))

    def dist_route_and_fold(self, records, fused) -> None:
        """records: CUDA tensor of fixed 64-byte records in arrival order carrying GLOBAL aggregate indices.
        fused: 0 NCCL all-to-all, 1 peer scatter, 2 pipelined push + fold, 3 the same with projected records (see sgr.h)."""
        r, nbytes = self._lend(records)
        self._ck(self._lib.sgr_dist_route_and_fold(self._h, r, nbytes // 64, int(fused)))

    def dist_recv_base(self) -> int:
        p = C.c_void_p()
        self._ck(self._lib.sgr_dist_recv_base(self._h, C.byref(p)))
        return int(p.value or 0)

    def dist_set_peers(self, bases: Sequence[int]) -> None:
        """Loopback ranks (one process, one device): the other ranks' receive allocations as raw device pointers."""
        arr = (C.c_void_p * len(bases))(*[C.c_void_p(b) for b in bases])
        self._ck(self._lib.sgr_dist_set_peers(self._h, arr))

    def dist_reserve(self, max_records: int) -> None:
        """Allocate everything the pipelined push needs up front (required for loopback ranks, see sgr.h)."""
        self._ck(self._lib.sgr_dist_reserve(self._h, int(max_records)))

    def states_hash(self) -> int:
        """Order-independent 64-bit hash of the live table (global aggregate indices on a routed engine)."""
        h = C.c_uint64()
        self._ck(self._lib.sgr_states_hash(self._h, C.byref(h)))
        return int(h.value)

    def dist_stats(self) -> N.sgr_dist_stats:
        s = N.sgr_dist_stats()
        self._ck(self._lib.sgr_dist_get_stats(self._h, C.byref(s)))
        return s

    def dist_local_aggregates(self) -> np.ndarray:
        n = C.c_uint64()
        self._ck(self._lib.sgr_dist_local_aggregates(self._h, None, 0, C.byref(n)))
        out = np.zeros(int(n.value), dtype=np.uint32)
        self._ck(self._lib.sgr_dist_local_aggregates(self._h, out.ctypes.data, len(out), C.byref(n)))
        return out

    def dist_load_keys(self, ids: Sequence) -> None:
        """The ids of global aggregates 0..n_global - 1 (str or bytes), in the partition table's order (sgr_dist_load_keys):
        this rank keeps the ones it owns, in local-slot order, and get(), get_many(), export_changes(), scan() and their
        *_values twins then read its rows by id. An id another rank owns is unknown here."""
        blob, offs = _id_batch([k if isinstance(k, bytes) else k.encode("utf-8") for k in ids])
        self._ck(self._lib.sgr_dist_load_keys(self._h, blob.ctypes.data, offs.ctypes.data, len(offs) - 1))

    def stats(self) -> N.sgr_stats:
        s = N.sgr_stats()
        self._ck(self._lib.sgr_get_stats(self._h, C.byref(s)))
        return s

    def set_option(self, name: str, value: int) -> None:
        """Engine options (include/sgr.h). Fold-source options: "head_plane" 0 keeps every fold on the log; "head_variant"
        -1 (the default) picks the slot plane where the program fits it, 0..4 keeps the 32-byte head plane with that kernel
        configuration; "proj_variant" picks the slot plane's kernel configuration."""
        self._ck(self._lib.sgr_set_option(self._h, name.encode(), int(value)))

    def stream_ptr(self) -> int:
        p = C.c_void_p()
        self._ck(self._lib.sgr_stream(self._h, C.byref(p)))
        return int(p.value or 0)

"""Restatement of sgr_put_batch (include/sgr.h) in NumPy: the KTable a state topic restores (SurgeStateStoreConsumer.scala:57-76,
last write wins per key, a null value deletes: SurgeModel.scala:62-64), written over the engine's table layout.

Table: `ids` (the key table, dense index = position), `states` u8[n_rows, state_bytes] (program bytes, then u32 flags, u32
err_idx). A batch is records in arrival order: (id, program bytes) or (id, None) for a tombstone. The result is what folding
each record as a snapshot event (CREATE + SET of every program byte) or a TOMBSTONE event gives, as one fold:
  * new ids get the next dense indices in order of first appearance (a tombstone of an unknown id too, with a None row);
  * the last record per id decides its row: its bytes with EXISTS, or None (program bytes zero, no EXISTS);
  * CHANGED compares the end state with the state before the batch, as a new instance: Double fields with == (NaN never
    equal, 0.0 == -0.0), every other word bitwise; a None state is equal only to None;
  * every row loses CHANGED and ERROR first and err_idx is 0 (the batch is "the last fold").
Never imported by surge_b200/."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

EXISTS, CHANGED, ERROR = 1, 2, 4


def _differ(new: np.ndarray, old: np.ndarray, f64_offsets: Sequence[int]) -> bool:
    f64_words = set()
    for off in f64_offsets:
        f64_words.update((off // 4, off // 4 + 1))
    nw, ow = new.view(np.uint32), old.view(np.uint32)
    for w in range(len(nw)):
        if w not in f64_words and nw[w] != ow[w]:
            return True
    for off in f64_offsets:
        x = new[off:off + 8].view(np.float64)[0]
        y = old[off:off + 8].view(np.float64)[0]
        if not (x == y):
            return True
    return False


def put_batch(ids: List[str], states: np.ndarray, batch: Sequence[Tuple[str, Optional[bytes]]],
              f64_offsets: Sequence[int] = ()) -> Tuple[List[str], np.ndarray, int]:
    """(key table, table, new ids) after one batch; the inputs are not modified. The table grows to the key table's size when
    it is shorter (new rows None)."""
    sb = states.shape[1]
    user = sb - 8
    ids = list(ids)
    index = {k: i for i, k in enumerate(ids)}
    n0 = len(ids)
    last = {}
    for pos, (k, _) in enumerate(batch):
        if k not in index:
            index[k] = len(ids)
            ids.append(k)
        last[index[k]] = pos
    out = np.zeros((max(len(states), len(ids)), sb), dtype=np.uint8)
    out[:len(states)] = states
    fl = out[:, user:user + 4].copy().view(np.uint32)[:, 0]
    fl &= EXISTS
    out[:, user:user + 4] = fl.astype(np.uint32).view(np.uint8).reshape(-1, 4)
    out[:, user + 4:] = 0
    for slot, pos in last.items():
        value = batch[pos][1]
        old_exists = bool(out[slot, user:user + 4].view(np.uint32)[0] & EXISTS)
        if value is not None:
            row = np.zeros(user, dtype=np.uint8)
            row[:len(value)] = np.frombuffer(value, dtype=np.uint8)
            changed = not old_exists or _differ(row, out[slot, :user].copy(), f64_offsets)
            flags = EXISTS | (CHANGED if changed else 0)
        else:
            row = np.zeros(user, dtype=np.uint8)
            flags = CHANGED if old_exists else 0
        out[slot, :user] = row
        out[slot, user:user + 4] = np.frombuffer(np.uint32(flags).tobytes(), dtype=np.uint8)
    return ids, out, len(ids) - n0

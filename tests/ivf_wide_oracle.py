"""numpy restatement of what the wide IVF searches (crag_ivf_search_i8_wide, crag_ivf_search_pq_wide) add to the narrow
ones, bit for bit: the slot order of a query's probed rows, clamped to max_probe_rows, and the map of slots back to
stored positions.  S1, the key order and the rescore are tests/ivf_i8_oracle.py's and tests/ivf_pq_oracle.py's, whose
search_i8 / search_pq take any n_cand; DESIGN.md section 7 states the semantics.

  probed lists  a query's probes in [0, nlist), each list once, in ascending list id (empty lists give no rows)
  slot order    the probed lists' real rows, list after list, stored order inside a list: slot s is the s-th of them
  clamp         only the first max_probe_rows slots are scored; stage 1 is the top n_cand of those by (S1 descending,
                slot ascending), and slot order is stored-position order, so that is (S1 descending, position
                ascending)

Test infrastructure only: the product path never imports this module.
"""
from __future__ import annotations

import numpy as np

from oracle import quant_oracle as qo

TILE_ROWS = 128


def probed_lists(probed_ids_row: np.ndarray, nlist: int) -> list:
    """A query's distinct valid probes in ascending list id."""
    return sorted({int(l) for l in np.asarray(probed_ids_row) if 0 <= l < nlist})


def slot_positions(probed_ids_row, list_tile_start, list_rows, nlist: int, max_probe_rows: int) -> np.ndarray:
    """Stored position of every scored slot of one query, in slot order (int64 [n_q])."""
    starts = np.asarray(list_tile_start, np.int64)
    rows = np.asarray(list_rows, np.int64)
    parts = [starts[l] * TILE_ROWS + np.arange(max(int(rows[l]), 0), dtype=np.int64)
             for l in probed_lists(probed_ids_row, nlist)]
    pos = np.concatenate(parts) if parts else np.zeros(0, np.int64)
    return pos[:max_probe_rows]


def stage1(s1: np.ndarray, positions: np.ndarray, n_cand: int):
    """The top n_cand of one query's scored slots: (slots [n_cand], positions [n_cand], S1 [n_cand]), -1 / -inf past
    n_q, and the (min, max) of S1 over them ((+inf, -inf) for none)."""
    s1 = np.asarray(s1, np.float32)
    slots = np.arange(s1.size, dtype=np.int64)
    top, sc = qo.topk_keys(s1, slots, n_cand)
    pos = np.where(top >= 0, positions[np.maximum(top, 0)] if positions.size else -1, -1)
    if s1.size:
        o = qo.orderable(s1)
        mm = np.array([s1[np.argmin(o)], s1[np.argmax(o)]], np.float32)
    else:
        mm = np.array([np.inf, -np.inf], np.float32)
    return top, pos.astype(np.int64), sc, mm

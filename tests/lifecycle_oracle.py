"""A model of a ``CorpusIndex`` that is changed many times (``insert_documents``, ``delete_documents``,
``delete_documents_by_metadata``, ``append``, ``delete_chunks``, ``compact``, ``add_tsvector_rows``): a list of chunk
records with their stored rows, an alive flag and a tsvector flag, changed by the reference's rules, and what the device
index must hold after each change.  NumPy only: a failing GPU program replays here step by step.

Rules (``raglite/_insert.py``, ``raglite/_delete.py``): duplicate document ids collapse to the last document given, blank
documents are dropped, documents with live chunks are skipped, a failing insert changes nothing; deletes count the
documents that had live chunks; metadata deletes match ``Document`` records only; ``compact`` drops the dead records and
renumbers the rest in order.  A float16 model widens to float32 where ``CorpusIndex.append`` does.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import Any

import numpy as np
import rounding as rd


@dataclass
class Record:
    id: str
    document_id: str
    index: int
    body: str
    metadata: dict[str, Any]
    rows: np.ndarray          # float32 [n, d]: the values stored (float16 values widened when storage is fp16)
    alive: bool = True
    tsvector: bool = False
    chunk: Any = None         # the Chunk record the device is expected to hold


def contains(metadata: dict[str, Any], flt: dict[str, Any]) -> bool:
    """JSON containment of a filter (values made lists) in list-valued metadata."""
    for k, want in flt.items():
        want = want if isinstance(want, list) else [want]
        have = metadata.get(k)
        if have is None:
            return False
        have = have if isinstance(have, (list, tuple)) else [have]
        if not all(w in have for w in want):
            return False
    return True


def unit_scale(rows: np.ndarray) -> bool:
    """The fp16 fast path's gate as ``rl_row_stats`` decides it: every row's float64 sum of squares s > 0, float32(1 /
    sqrt(s)) <= 2, every |x| <= 1024.  (Exact for float16 values, whose squares are multiples of 2^-48.)"""
    if rows.size == 0:
        return False
    r64 = rows.astype(np.float64)
    s = np.einsum("ij,ij->i", r64, r64)
    with np.errstate(divide="ignore"):
        inv = (1.0 / np.sqrt(s)).astype(np.float32)
    return bool((s > 0).all() and (inv <= 2.0).all() and np.abs(rows).max() <= 1024)


def fp16_exact(rows: np.ndarray) -> bool:
    with np.errstate(over="ignore"):
        return bool(np.array_equal(rows.astype(np.float16).astype(np.float32), rows))


class Model:
    def __init__(self, storage: str, d: int) -> None:
        self.storage, self.d = storage, d
        self.records: list[Record] = []
        self.documents: dict[str, Any] = {}      # Document records insert_documents kept, by id
        self.has_tsrank = False                  # add_tsvector_rows has been called once

    # ---- operations -------------------------------------------------------------------------------------------------
    def live_document_ids(self) -> set[str]:
        return {r.document_id for r in self.records if r.alive}

    def insert(self, documents: list[Any], records_of: Any, *, fail: bool = False) -> list[Any]:
        """``insert_documents``: ``records_of(doc) -> list[Record]`` gives a document's chunks and rows.  Returns the
        documents actually inserted, in order.  ``fail``: processing raises, nothing changes."""
        if not all(isinstance(doc.content, str) for doc in documents):
            raise ValueError("Some or all documents have missing `document.content`.")
        docs = [doc for doc in {doc.id: doc for doc in documents}.values() if doc.content.strip()]
        present = self.live_document_ids()
        docs = [doc for doc in docs if doc.id not in present]
        if not docs or fail:
            return []
        recs = [r for doc in docs for r in records_of(doc)]
        self._append(recs)
        self.documents.update({doc.id: doc for doc in docs})
        return docs

    def append(self, recs: list[Record]) -> None:
        """``CorpusIndex.append``: a chunk id that is alive already is refused."""
        live = {r.id for r in self.records if r.alive}
        if any(r.id in live for r in recs):
            raise ValueError("already in the index")
        self._append(recs)

    def _append(self, recs: list[Record]) -> None:
        if not recs:
            return
        new = np.concatenate([r.rows for r in recs])
        if self.storage == "fp16":
            resident = self.resident_rows()
            ok = len(resident) == 0 or unit_scale(resident)
            if not fp16_exact(new) or (ok and not unit_scale(new)):
                self.storage = "fp32"
        self.records += recs

    def delete_documents(self, ids: list[str]) -> int:
        present = self.live_document_ids() & set(ids)
        for r in self.records:
            if r.document_id in present:
                r.alive = False
        for i in present:
            self.documents.pop(i, None)
        return len(present)

    def delete_by_metadata(self, flt: dict[str, Any]) -> int:
        return self.delete_documents([d.id for d in self.documents.values() if contains(d.metadata_, flt)])

    def delete_chunks(self, ids: list[str]) -> int:
        n = 0
        for r in self.records:
            if r.alive and r.id in set(ids):
                r.alive, n = False, n + 1
        return n

    def compact(self) -> None:
        self.records = [r for r in self.records if r.alive]

    def add_tsvectors(self, ids: list[str]) -> list[Record]:
        """The records ``add_tsvector_rows`` marks: the last record of each id."""
        last = {r.id: r for r in self.records}
        out = [last[i] for i in ids]
        if any(r.tsvector for r in out):
            raise ValueError("already has a tsvector")
        for r in out:
            r.tsvector = True
        self.has_tsrank = True
        return out

    # ---- what the device must hold ------------------------------------------------------------------------------------
    def counts(self) -> np.ndarray:
        return np.asarray([len(r.rows) for r in self.records], np.int64)

    def chunk_off(self) -> np.ndarray:
        return np.concatenate([[0], np.cumsum(self.counts())]).astype(np.int64)

    def row_chunk(self) -> np.ndarray:
        return np.repeat(np.arange(len(self.records), dtype=np.int32), self.counts())

    def chunk_alive(self) -> np.ndarray:
        return np.asarray([r.alive for r in self.records], bool)

    def row_alive(self) -> np.ndarray:
        return np.repeat(self.chunk_alive(), self.counts())

    def resident_rows(self) -> np.ndarray:
        return np.concatenate([r.rows for r in self.records]) if self.records else np.zeros((0, self.d), np.float32)

    def live(self) -> list[Record]:
        return [r for r in self.records if r.alive]

    def rows_unit_scale(self) -> bool:
        """``rows_unit_scale``: statistics over every resident row, tombstoned ones included (compact drops them)."""
        return unit_scale(self.resident_rows())

    def n_live_rows(self) -> int:
        return int(sum(len(r.rows) for r in self.live()))


def check_row_stats(X: np.ndarray, inv: np.ndarray, sq: np.ndarray, st: np.ndarray | None, tag: str) -> None:
    """``rl_row_stats`` outputs for rows X (as stored) against float64, with the kernel's bound as
    ``test_gpu_index_kernels._check_row_stats`` states it: the sum of squares exact where every partial sum is (a
    multiple of the smallest square below 2^53 of them), else within 2 gamma_{d-1} S; 1/|e| and max |e| within 2
    gamma_{d+4} of their value.  ``st`` (or None) the statistics over the same rows."""
    d = X.shape[1]
    X64 = X.astype(np.float64)
    S = np.einsum("ij,ij->i", X64, X64)
    A = np.abs(X)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = np.where(A > 0, np.spacing(A).astype(np.float64), np.inf).min(axis=1)
        bound = np.where(S < 2.0 ** 53 * m * m, 0.0, 2 * rd.gamma(d - 1) * S)
        inv_v = np.where(S > 0, 1.0 / np.sqrt(S), 0.0)
    rd.check(sq, S, bound, rd.f32, what=f"sq_norm {tag}")
    rd.check(inv, inv_v, 2 * rd.gamma(d + 4) * inv_v, rd.f32, what=f"inv_norm {tag}")
    if st is None or len(X) == 0:
        return
    nmax = np.sqrt(S.max())
    rd.check(st[0], nmax, 2 * rd.gamma(d + 4) * nmax, rd.f32, what=f"stats[0] {tag}")
    assert st[1] == np.float32(A.max()), (tag, st[1])
    nz = S > 0
    imax = 1.0 / np.sqrt(S[nz].min()) if nz.any() else 0.0
    rd.check(st[2], imax, 2 * rd.gamma(d + 4) * imax, rd.f32, what=f"stats[2] {tag}")
    assert st[3] == (0.0 if nz.all() else 1.0), (tag, st[3])


# ---- planted float16 rows at the fp16 gate ---------------------------------------------------------------------------
def fp16_row_with_sum_sq(target: float, d: int) -> np.ndarray:
    """A float16 row of width d whose exact float64 sum of squares is ``target`` (a multiple of 2^-48 below 1): the
    greedy largest float16 square that still fits, until nothing is left."""
    row = np.zeros(d, np.float16)
    left = float(target)
    for j in range(d):
        if left == 0:
            break
        c = np.float16(np.sqrt(left))
        while float(c) ** 2 > left:
            c = np.nextafter(c, np.float16(0))
        if c == 0:
            break
        row[j] = c
        left -= float(c) ** 2
    assert left == 0, (target, left)
    return row


def planted_gate_rows(d: int) -> dict[str, np.ndarray]:
    """Float16 rows at the edges of the gate: norms of 0.5 minus and plus one float32 ulp, exactly 0.5, the sum of
    squares one float32 step below 0.25 (which float32 1/sqrt rounds back to 2), |x| = 1024 and 1025, a zero row."""
    half = 0.5
    rows = {
        "norm 0.5 - 1 ulp": fp16_row_with_sum_sq(round((half - 2.0 ** -25) ** 2 * 2.0 ** 48) / 2.0 ** 48, d),
        "norm 0.5": fp16_row_with_sum_sq(0.25, d),
        "norm 0.5 + 1 ulp": fp16_row_with_sum_sq(round((half + 2.0 ** -24) ** 2 * 2.0 ** 48) / 2.0 ** 48, d),
        "sum sq 0.25 - 2^-26": fp16_row_with_sum_sq(0.25 - 2.0 ** -26, d),
        "sum sq 0.25 - 2^-24": fp16_row_with_sum_sq(0.25 - 2.0 ** -24, d),
    }
    for big in (1024.0, 1025.0):
        r = np.zeros(d, np.float16)
        r[d // 2] = big
        r[1] = 0.75
        rows[f"|x| = {big:g}"] = r
    rows["zero"] = np.zeros(d, np.float16)
    return rows

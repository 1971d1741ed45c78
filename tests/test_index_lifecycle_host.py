"""The lifecycle model's own rules (``tests/lifecycle_oracle.py``) and the float16 rows it plants at the storage gate,
on the CPU: dedup, skip, blank documents, atomic failure, delete counts, metadata deletes, compact renumbering, widening;
the planted rows' exact sums of squares, and the host gate of ``CorpusIndex._pick_storage`` deciding as the model's
restatement of ``rl_row_stats_f16`` does."""

from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any

import lifecycle_oracle as lo
import numpy as np
import pytest

from raglite_b200._index import CorpusIndex, fp16_rows_unit_scale


@dataclass
class Doc:
    id: str
    content: str | None
    metadata_: dict[str, Any] = field(default_factory=dict)


def _records(doc: Doc) -> list[lo.Record]:
    n = 1 + len(doc.content) % 3
    rows = np.ones((1, 8), np.float32) * np.float32(0.5)
    return [lo.Record(f"{doc.id}-{i}:{doc.content}"[:40], doc.id, i, doc.content, dict(doc.metadata_), rows.copy())
            for i in range(n)]


def test_insert_rules():
    m = lo.Model("fp32", 8)
    a, a2, b, blank = Doc("a", "first"), Doc("a", "second!"), Doc("b", "bee"), Doc("c", "  \n ")
    assert [d.content for d in m.insert([a, b, a2, blank], _records)] == ["second!", "bee"]   # last one of an id wins
    assert {r.document_id for r in m.live()} == {"a", "b"} and set(m.documents) == {"a", "b"}
    assert m.insert([a, Doc("b", "other")], _records) == []                                    # live documents: skipped
    before = [r.id for r in m.records]
    assert m.insert([Doc("d", "dee")], _records, fail=True) == [] and [r.id for r in m.records] == before
    with pytest.raises(ValueError, match="missing"):
        m.insert([Doc("e", None)], _records)


def test_deletes_count_documents_with_live_chunks():
    m = lo.Model("fp32", 8)
    m.insert([Doc("a", "x", {"topic": ["t1"]}), Doc("b", "yy", {"topic": ["t2"]}), Doc("c", "zzz", {"topic": ["t1"]})],
             _records)
    m.append([lo.Record("s0", "synthetic", 0, "", {"topic": ["t1"]}, np.ones((2, 8), np.float32))])
    assert m.delete_documents(["a", "a", "nope"]) == 1 and m.delete_documents(["a"]) == 0
    assert m.delete_by_metadata({"topic": "t1"}) == 1                     # "c"; the synthetic chunk has no Document
    assert {r.document_id for r in m.live()} == {"b", "synthetic"}
    assert m.delete_chunks(["s0", "s0", "unknown"]) == 1 and m.delete_chunks(["s0"]) == 0
    assert m.delete_documents(["synthetic"]) == 0


def test_reinsert_compact_renumbers_and_keeps_the_live_copy():
    m = lo.Model("fp32", 8)
    a = Doc("a", "text")
    m.insert([a, Doc("b", "more")], _records)
    n_a = sum(1 for r in m.records if r.document_id == "a")
    for _ in range(2):
        assert m.delete_documents(["a"]) == 1
        assert m.insert([a], _records) == [a]
    assert len(m.records) == 3 * n_a + sum(1 for r in m.records if r.document_id == "b")
    dead = [i for i, r in enumerate(m.records) if not r.alive]
    assert len(dead) == 2 * n_a and m.chunk_alive().sum() == len(m.records) - 2 * n_a
    with pytest.raises(ValueError, match="already"):
        m.append([m.live()[0]])
    assert m.add_tsvectors([m.records[0].id])[0] is m.records[-n_a]       # the last copy of an id
    m.compact()
    assert all(r.alive for r in m.records) and [r.document_id for r in m.records].count("a") == n_a
    np.testing.assert_array_equal(m.chunk_off(), np.concatenate([[0], np.cumsum(m.counts())]))
    np.testing.assert_array_equal(m.row_chunk(), np.repeat(np.arange(len(m.records)), m.counts()))
    assert m.records[-n_a].tsvector and not m.records[-1].tsvector


def test_widening_follows_the_gate_of_the_resident_rows():
    planted = lo.planted_gate_rows(64)
    unit = np.full((1, 64), 0.125, np.float32)                           # norm 1
    m = lo.Model("fp16", 64)
    m.append([lo.Record("u", "d", 0, "", {}, unit)])
    m.append([lo.Record("n", "d", 1, "", {}, planted["norm 0.5"].astype(np.float32)[None])])
    assert m.storage == "fp16" and m.rows_unit_scale()
    m.append([lo.Record("z", "d", 2, "", {}, planted["zero"].astype(np.float32)[None])])
    assert m.storage == "fp32" and not m.rows_unit_scale()
    m = lo.Model("fp16", 64)
    m.append([lo.Record("x", "d", 0, "", {}, unit + np.float32(1e-4))])   # not a float16 value
    assert m.storage == "fp32"


def test_planted_rows_sit_on_the_gate():
    for d in (64, 1024):
        rows = lo.planted_gate_rows(d)
        s = {k: float((r.astype(np.float64) ** 2).sum()) for k, r in rows.items()}
        assert s["norm 0.5"] == 0.25 and s["zero"] == 0.0
        assert np.float32(np.sqrt(s["norm 0.5 - 1 ulp"])) == np.nextafter(np.float32(0.5), np.float32(0))
        assert np.float32(np.sqrt(s["norm 0.5 + 1 ulp"])) == np.nextafter(np.float32(0.5), np.float32(1))
        assert s["sum sq 0.25 - 2^-26"] == 0.25 - 2.0 ** -26
        decide = {k: lo.unit_scale(r[None].astype(np.float32)) for k, r in rows.items()}
        assert decide == {"norm 0.5 - 1 ulp": False, "norm 0.5": True, "norm 0.5 + 1 ulp": True,
                          "sum sq 0.25 - 2^-26": True, "sum sq 0.25 - 2^-24": False, "|x| = 1024": True,
                          "|x| = 1025": False, "zero": False}
        for k, r in rows.items():
            assert fp16_rows_unit_scale(r[None]) == decide[k], k
            want = "fp16" if decide[k] else "fp32"
            assert CorpusIndex._pick_storage(np.stack([r, rows["norm 0.5"]]).astype(np.float32), "auto")[1] == want, k
        # the float32 norm a host gate could compare with 0.5 refuses a row the device's float32 1/sqrt accepts
        assert np.linalg.norm(rows["sum sq 0.25 - 2^-26"].astype(np.float32)) < 0.5 and decide["sum sq 0.25 - 2^-26"]

"""Ingest on the host: ``Document.from_text`` / ``from_path``, the heading rules and chunk records against
``insert_oracle`` and hand-written expectations, the rules ``insert_documents`` applies before any device work (content
check, duplicates, blanks, documents already in the index, a sharded index, the failure wrapper), the empty-filter
error, and the argument checks of ``rl_chunk_embedding_blend`` before any CUDA call."""

from __future__ import annotations

import ctypes as C

import insert_oracle as io
import numpy as np
import pytest

import raglite_b200 as rl
from raglite_b200 import _insert as I  # noqa: N812

RL_EINVAL, RL_EUNSUPPORTED = -1, -4


# ---- documents -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("content, kw", [
    ("# Title\n\nBody text.", {}),
    ("\n\n   \n  First line after blanks  \nsecond", {}),
    ("x" * 81 + "\nrest", {}),
    ("y" * 80 + "\nrest", {}),
    ("Ünïcödé ✓ content", {"url": "https://example.org/a", "filename": "given.md", "topic": ["a", "b"], "year": 2024}),
    ("Same", {"id": "my-id", "tags": ("t",)}),
])
def test_document_from_text(content, kw):
    doc = rl.Document.from_text(content, **kw)
    want = io.document_fields(content, **kw)
    assert (doc.id, doc.filename, doc.url, doc.metadata_, doc.content) == tuple(want[k] for k in (
        "id", "filename", "url", "metadata_", "content"))


def test_document_from_text_hand_values():
    doc = rl.Document.from_text("\n\n  " + "z" * 90 + "  \nmore")
    assert doc.filename == "z" * 80 + "..." and doc.id == io.sha16("\n\n  " + "z" * 90 + "  \nmore")
    assert doc.metadata_ == {"filename": [doc.filename], "uri": [None], "url": [None], "size": [len(doc.content)]}
    assert rl.Document.from_text("é").metadata_["size"] == [2]
    assert rl.Document.from_text("a", id="x").metadata_["uri"] == ["x"]


def test_document_from_path(tmp_path):
    p = tmp_path / "notes.md"
    p.write_text("# Notes\n\nSome text.\n")
    doc = rl.Document.from_path(p, url="u", lang="en")
    assert doc.id == io.sha16("# Notes\n\nSome text.\n") and doc.filename == "notes.md" and doc.content == p.read_text()
    st = p.stat()
    assert doc.metadata_ == {"filename": ["notes.md"], "uri": [None], "url": ["u"], "size": [st.st_size],
                             "created": [st.st_ctime], "modified": [st.st_mtime], "lang": ["en"]}
    t = tmp_path / "a.txt"
    t.write_text("plain")
    assert rl.Document.from_path(t, id="given").id == "given"
    pdf = tmp_path / "a.pdf"
    pdf.write_bytes(b"%PDF")
    with pytest.raises(ValueError, match="only .md and .txt"):
        rl.Document.from_path(pdf)


# ---- headings ----------------------------------------------------------------------------------------------------------
HEADING_CASES = {
    "atx": ("# A\n\ntext\n\n## B\n\n### C\n\nmore\n\n## D\n", ["# A", "## D", "", "", "", ""]),
    "setext": ("Top\n===\n\npara\n\nSub\n---\n", ["# Top", "## Sub", "", "", "", ""]),
    "fence_and_quote": ("# Real\n\n```\n# not a heading\n```\n\n> ## quoted\n\n    # indented code\n",
                        ["# Real", "## quoted", "", "", "", ""]),
    "newlines": ("Line one\nline two\n===\n\n#### deep   \n", ["# Line one line two", "", "", "#### deep", "", ""]),
    "closing_hashes": ("## Two ##\n\n###### Six\n", ["", "## Two", "", "", "", "###### Six"]),
    "empty": ("", ["", "", "", "", "", ""]),
}


@pytest.mark.parametrize("name", sorted(HEADING_CASES))
def test_heading_lines(name):
    doc, want = HEADING_CASES[name]
    assert I.extract_heading_lines(doc) == io.heading_lines(doc) == want


@pytest.mark.parametrize("doc, want", [
    ("# A\n\n## B\n\ntext\n\n### C\n", ["# A", "## B", "", "", "", ""]),   # stops at the first non-heading text
    ("\n\n## B\n\n# A\n", ["# A", "", "", "", "", ""]),
    ("text first\n\n# A\n", ["", "", "", "", "", ""]),
    ("```\ncode\n```\n\n# A\n", ["", "", "", "", "", ""]),                 # a fence has content: the scan stops
    ("> # quoted\n\n## B\n", ["# quoted", "## B", "", "", "", ""]),
])
def test_heading_lines_leading_only(doc, want):
    assert I.extract_heading_lines(doc, leading_only=True) == io.heading_lines(doc, leading_only=True) == want


@pytest.mark.parametrize("headings, body, want", [
    ("# A\n## B\n### C", "plain body", "# A\n## B\n### C"),
    ("# A\n## B\n### C", "## New\n\nbody", "# A"),            # a body opening at a higher level than the deepest
    ("# A\n## B", "#### Deep\n\nbody", "# A\n## B"),          # ... or at a lower one
    ("# A\n## B", "# Other\n\nbody", ""),
    ("# A\n## B", "body\n\n# Late", "# A\n## B"),             # a heading after text does not truncate
    ("", "## X\n\nbody", ""),
])
def test_truncate_headings(headings, body, want):
    assert I.truncate_headings(headings, body) == io.truncated(headings, body) == want


def test_chunk_records_and_front_matter():
    doc = rl.Document.from_text("# Guide\n\nIntro.\n\n## Part\n\nText.\n\n# Next\n\nEnd.", filename="guide.md",
                                url="https://x.org", topic="t")
    bodies = ["# Guide\n\nIntro.\n\n", "## Part\n\nText.\n\n", "More text.\n\n", "# Next\n\nEnd."]
    got = I.chunk_records(doc, bodies)
    assert got == io.records(doc.id, doc.filename, doc.url, doc.metadata_, bodies)
    assert [c.id for c in got] == [io.sha16(f"{doc.id}-{i}") for i in range(4)]
    assert [c.headings for c in got] == ["", "# Guide", "# Guide\n## Part", ""]
    assert [c.index for c in got] == [0, 1, 2, 3] and all(c.document_id == doc.id for c in got)
    # the document's metadata (list-valued filename included) overrides the record's own filename / url
    assert got[0].metadata_ == {"filename": ["guide.md"], "url": ["https://x.org"], "uri": [None], "size": [len(doc.content)],
                                "topic": ["t"]}
    assert got[2].front_matter == "---\nfilename: ['guide.md']\nurl: ['https://x.org']\nuri: [None]\n---"
    assert got[2].content == got[2].front_matter + "\n\n# Guide\n## Part\n\nMore text."
    plain = I.chunk_from_body(rl.Document(id="d", filename="f"), 0, "body")
    assert plain.metadata_ == {"filename": ["f"], "url": [None]} and plain.front_matter == "---\nfilename: ['f']\nurl: [None]\n---"


# ---- insert_documents' rules before any device work -----------------------------------------------------------------------
class _Stop(Exception):
    pass


@pytest.fixture
def captured(monkeypatch):
    """Stops insert_documents where the device work would begin, keeping the documents it would process."""
    seen: list[list[str]] = []

    def groups(docs, config):  # noqa: ANN001, ANN202
        seen.append([d.id for d in docs])
        raise _Stop("stopped")

    monkeypatch.setattr(I, "_document_groups", groups)
    return seen


def _cfg(name: str) -> rl.RAGLiteConfig:
    return rl.RAGLiteConfig(db_url=f"host-test://{name}", reranker=None)


def test_content_required_and_blank_documents(captured):
    cfg = _cfg("content")
    with pytest.raises(ValueError, match="missing `document.content`"):
        rl.insert_documents([rl.Document.from_text("a"), rl.Document(id="x", filename="x")], config=cfg)
    rl.insert_documents([rl.Document.from_text("   \n\t "), rl.Document.from_text("")], config=cfg)
    rl.insert_documents([], config=cfg)
    assert captured == [] and rl.get_index(cfg) is None


def test_duplicates_collapse_in_input_order_and_failures_wrap(captured):
    cfg = _cfg("dedup")
    a1, b, a2 = (rl.Document.from_text("one", id="a"), rl.Document.from_text("two", id="b"),
                 rl.Document.from_text("three", id="a"))
    c, blank = rl.Document.from_text("four", id="c"), rl.Document.from_text("  ", id="z")
    with pytest.raises(ValueError, match="Error processing document: stopped") as e:
        rl.insert_documents([a1, b, blank, a2, c], config=cfg)
    assert isinstance(e.value.__cause__, _Stop)
    assert captured == [["a", "b", "c"]]
    assert rl.get_index(cfg) is None


def _host_index(chunks: list[rl.Chunk], alive: list[bool]) -> rl.CorpusIndex:
    """A CorpusIndex shell holding only the host tables the insert rules read."""
    idx = rl.CorpusIndex.__new__(rl.CorpusIndex)
    idx.chunks, idx.chunk_ids, idx.chunk_metadata = chunks, [c.id for c in chunks], [c.metadata_ for c in chunks]
    idx.n_chunks, idx._chunk_alive, idx.documents = len(chunks), np.asarray(alive, dtype=bool), {}
    return idx


def test_documents_with_live_chunks_are_skipped(captured):
    cfg = _cfg("skip")
    chunks = [rl.Chunk(id="c0", document_id="a"), rl.Chunk(id="c1", document_id="b"), rl.Chunk(id="c2", document_id="b")]
    rl.register_index(cfg, _host_index(chunks, [True, False, False]))
    try:
        rl.insert_documents([rl.Document.from_text("x", id="a")], config=cfg)          # all present: nothing to do
        assert captured == []
        with pytest.raises(ValueError, match="Error processing document"):
            rl.insert_documents([rl.Document.from_text("x", id=i) for i in "abc"], config=cfg)
        assert captured == [["b", "c"]]                                               # b's chunks are deleted
    finally:
        rl.unregister_index(cfg)


def test_index_without_records_is_refused(captured):
    cfg = _cfg("bare")
    idx = _host_index([rl.Chunk(id="c0", document_id="a")], [True])
    idx.chunks = None
    rl.register_index(cfg, idx)
    try:
        with pytest.raises(ValueError, match="does not hold chunk ids, Chunk records"):
            rl.insert_documents([rl.Document.from_text("x")], config=cfg)
        assert captured == []
    finally:
        rl.unregister_index(cfg)


def test_sharded_index_is_named():
    from raglite_b200._dist import ShardedIndex

    cfg = _cfg("sharded")
    rl.register_index(cfg, ShardedIndex.__new__(ShardedIndex))
    try:
        for call in (lambda: rl.insert_documents([rl.Document.from_text("x")], config=cfg),
                     lambda: rl.delete_documents(["x"], config=cfg),
                     lambda: rl.delete_documents_by_metadata({"k": "v"}, config=cfg)):
            with pytest.raises(NotImplementedError, match="ShardedIndex is registered"):
                call()
    finally:
        rl.unregister_index(cfg)


def test_delete_rules_on_the_host():
    cfg = _cfg("delete")
    with pytest.raises(ValueError, match="^metadata_filter cannot be empty to prevent accidental deletion of all documents$"):
        rl.delete_documents_by_metadata({}, config=cfg)
    assert rl.delete_documents([], config=cfg) == 0 and rl.delete_documents(["a"], config=cfg) == 0
    assert rl.delete_documents_by_metadata({"k": "v"}, config=cfg) == 0


@pytest.mark.parametrize("flt", [{"topic": "a"}, {"topic": ["a", "b"]}, {"topic": ["a", "c"]}, {"year": 2024},
                                 {"year": [2024], "topic": "b"}, {"missing": None}, {"url": None}, {"topic": []}])
def test_metadata_containment(flt):
    docs = [rl.Document.from_text("x", topic=["a", "b"], year=2024), rl.Document.from_text("y", topic="a"),
            rl.Document.from_text("z", url="u")]
    got = [I.metadata_contains(d.metadata_, I.adapt_metadata(flt)) for d in docs]
    assert got == [io.contains(d.metadata_, flt) for d in docs]


# ---- rl_chunk_embedding_blend's argument checks --------------------------------------------------------------------------
def test_blend_refusals():
    from raglite_b200 import _lib

    lib = _lib.load()
    p = C.c_void_p(256)

    def blend(X=p, ldx=64, F=p, off=p, C_=3, N=10, d=64, out=p):  # noqa: N803
        return lib.rl_chunk_embedding_blend(X, ldx, F, off, C_, N, d, 12493, 15053, out, None)

    for bad in (dict(N=-1), dict(C_=-1), dict(d=0), dict(ldx=56), dict(C_=0)):
        assert blend(**bad) == RL_EINVAL, bad
        assert "bad shape" in lib.rl_last_error().decode()
    for bad in (dict(d=60, ldx=64), dict(ldx=68), dict(X=C.c_void_p(264)), dict(F=C.c_void_p(260)),
                dict(out=C.c_void_p(258))):
        assert blend(**bad) == RL_EUNSUPPORTED, bad
        assert "16-byte aligned" in lib.rl_last_error().decode()
    for k in ("X", "F", "off", "out"):
        assert blend(**{k: None}) == RL_EINVAL, k
        assert "null pointer" in lib.rl_last_error().decode()
    assert blend(N=0, C_=0, X=None, F=None, off=None, out=None) == 0


def test_blend_weights_are_weak_scalar_halves():
    a, b = (int(np.float16(w).view(np.uint16)) for w in (I.ALPHA, 1 - I.ALPHA))
    assert (a, b) == (12493, 15053)
    e = np.float16([1.0])
    assert (I.ALPHA * e).dtype == np.float16 and ((1 - I.ALPHA) * e)[0] == np.float16(1 - 0.15)


def test_numpy_blend_equals_the_float32_statement():
    """On this NumPy, ``α * e + (1 - α) * f`` on float16 rows is float16 and equals each product and the sum computed in
    float32 and rounded to float16, bit for bit (the GPU tests compare the kernel with the explicit statement)."""
    rng = np.random.default_rng(3)
    for scale in (1.0, 1e-4, 300.0):
        e, f = ((rng.standard_normal((200, 64)) * scale).astype(np.float16) for _ in range(2))
        got, want = io.blend_numpy(e, f), io.blend_f32(e, f)
        assert got.dtype == np.float16
        np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))

"""Generate golden vectors by running the REFERENCE's own code (dev container only).

Usage (needs /root/reference, which does not exist on the GPU box):

    python tools/make_golden_from_reference.py

``import raglite`` fails offline (duckdb/sqlalchemy/litellm/rerankers/llama_cpp are not
installed), but two pieces of the hot path are pure NumPy/SciPy once their imports resolve:

* ``raglite/_embed.py``  -- ``embed_strings_with_late_chunking`` / ``_embed_string_batch``
  (token counting, segmenting, largest-remainder split, mean pool, normalise, fp16 cast);
* ``raglite/_query_adapter.py`` -- ``_optimize_query_target``;
* ``raglite/_typing.py`` -- the column processors of the ``chunk_embedding.embedding`` column
  (DuckDB ``FLOAT[d]`` lists, PostgreSQL ``halfvec`` text, ``np.save`` blobs);
* ``raglite/_split_sentences.py`` -- ``split_sentences`` and ``markdown_sentence_boundaries``, with wtpsplit-lite's
  ``SaT`` replaced by a fake that returns seeded float32 probabilities;
* ``raglite/_split_chunklets.py`` and ``raglite/_split_chunks.py`` -- ``split_chunklets`` (with its Markdown boundaries
  and statement counts) and ``split_chunks`` (with the cost vector it hands to ``linprog``);
* ``raglite/_chatml_function_calling.py`` -- the chat handler's jinja template rendered on seeded message lists, and
  the handler itself run over a scripted ``Llama`` that records each completion's prompt, grammar and settings
  (``tests/golden/chatml_tools.json``).

This script loads those two files *unmodified from where they lie* under a synthetic ``raglite``
package whose heavy dependencies are replaced by stubs, and whose embedder is
``tests/fake_llama.FakeLlama``.  Outputs go to ``tests/golden/*.npz`` (committed).
"""

from __future__ import annotations

import importlib.util
import json
import sys
import types
from dataclasses import dataclass
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
REF = Path("/root/reference/src/raglite")
sys.path.insert(0, str(REPO / "tests"))
from fake_llama import FakeLlama, make_sentences  # noqa: E402

GOLDEN = REPO / "tests" / "golden"


class _Anything:
    """Attribute sink: any attribute / call returns another sink (for unused ORM symbols)."""

    def __getattr__(self, name):  # noqa: ANN001, ANN204
        return _Anything()

    def __call__(self, *a, **k):  # noqa: ANN002, ANN003, ANN204
        return _Anything()


def _stub(name: str, **attrs) -> types.ModuleType:  # noqa: ANN003
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)
    mod.__getattr__ = lambda attr: _Anything()  # type: ignore[method-assign]
    sys.modules[name] = mod
    return mod


def _load(name: str, path: Path) -> types.ModuleType:
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


@dataclass(frozen=True)
class _Config:
    embedder: str = "llama-cpp-python/fake/fake.gguf@64"
    embedder_normalize: bool = True
    vector_search_distance_metric: str = "cosine"


_CURRENT: dict[str, FakeLlama] = {}


class _LlamaCppPythonLLM:
    @staticmethod
    def llm(model: str, **kwargs):  # noqa: ANN003, ANN205, ARG004
        return _CURRENT["llm"]


def install_reference_stubs() -> tuple[types.ModuleType, types.ModuleType]:
    pkg = types.ModuleType("raglite")
    pkg.__path__ = []  # a package, but never executes the reference's __init__ (it imports the world)
    sys.modules["raglite"] = pkg
    _stub("litellm", embedding=_Anything())
    _stub("sqlalchemy", text=_Anything())
    _stub("sqlalchemy.orm")
    _stub("sqlalchemy.orm.attributes", flag_modified=_Anything())
    _stub("sqlmodel", Session=_Anything(), col=_Anything(), select=_Anything())
    _stub("raglite._config", RAGLiteConfig=_Config)
    _stub("raglite._lazy_llama", LLAMA_POOLING_TYPE_NONE=0, Llama=FakeLlama)
    _stub("raglite._litellm", LlamaCppPythonLLM=_LlamaCppPythonLLM)
    _stub("raglite._typing", FloatMatrix=np.ndarray, FloatVector=np.ndarray, IntVector=np.ndarray)
    _stub("raglite._database")
    _stub("raglite._search", vector_search=_Anything())
    embed = _load("raglite._embed", REF / "_embed.py")
    qa = _load("raglite._query_adapter", REF / "_query_adapter.py")
    return embed, qa


def golden_pool(embed_mod: types.ModuleType) -> None:
    cases = [
        dict(name="pool_small", n_sent=9, n_ctx=64, dim=32, seed=1, normalize=True),
        dict(name="pool_multi", n_sent=70, n_ctx=96, dim=48, seed=2, normalize=True),
        dict(name="pool_nonorm", n_sent=33, n_ctx=80, dim=40, seed=3, normalize=False),
        dict(name="pool_wide", n_sent=120, n_ctx=512, dim=384, seed=4, normalize=True),
    ]
    for c in cases:
        llm = FakeLlama(n_ctx=c["n_ctx"], dim=c["dim"], seed=c["seed"])
        _CURRENT["llm"] = llm
        sentences = make_sentences(c["n_sent"], seed=c["seed"])
        cfg = _Config(embedder_normalize=c["normalize"])
        out = embed_mod.embed_strings_with_late_chunking(sentences, config=cfg)
        simple = embed_mod._embed_string_batch(sentences[:7], config=cfg)  # noqa: SLF001
        np.savez_compressed(
            GOLDEN / f"{c['name']}.npz",
            meta=np.frombuffer(json.dumps({**c, "sentences": sentences}).encode(), dtype=np.uint8),
            late_chunking=out,
            simple=simple,
        )
        print(c["name"], out.shape, out.dtype, simple.shape)


def golden_adapter(qa_mod: types.ModuleType) -> None:
    rng = np.random.default_rng(7)
    arrays = {}
    for i, (d, npos, nneg, dtype) in enumerate([(16, 2, 5, np.float16), (48, 3, 9, np.float32), (96, 1, 12, np.float16)]):
        def unit(n):  # noqa: ANN001, ANN202
            x = rng.standard_normal((n, d))
            return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(dtype)
        q, P, N = unit(1)[0], unit(npos), unit(nneg)
        t = qa_mod._optimize_query_target(q, P, N, α=0.05)  # noqa: SLF001
        arrays.update({f"q{i}": q, f"P{i}": P, f"N{i}": N, f"t{i}": t})
    np.savez_compressed(GOLDEN / "adapter_target.npz", **arrays)
    print("adapter_target", sorted(arrays))


class _Generic:
    """Stand-in for SQLAlchemy's generic base classes (``TypeDecorator[...]``, ``UserDefinedType[...]``)."""

    Comparator: type

    def __class_getitem__(cls, item):  # noqa: ANN001, ANN206
        return cls

    def __init__(self, *a, **k) -> None:  # noqa: ANN002, ANN003
        pass


_Generic.Comparator = _Generic


def load_reference_typing() -> types.ModuleType:
    """``raglite/_typing.py`` unmodified, with SQLAlchemy reduced to the few names its class bodies touch:
    the column processors (``bind_processor`` / ``result_processor`` / ``process_*``) are pure NumPy."""
    for name in ("sqlalchemy", "sqlalchemy.engine", "sqlalchemy.ext", "sqlalchemy.ext.compiler", "sqlalchemy.sql",
                 "sqlalchemy.sql.functions", "sqlalchemy.sql.operators", "sqlalchemy.types"):
        _stub(name)
    sys.modules["sqlalchemy.ext.compiler"].compiles = lambda *a, **k: (lambda fn: fn)
    sys.modules["sqlalchemy.sql.functions"].FunctionElement = _Generic
    sys.modules["sqlalchemy.engine"].Dialect = object
    sys.modules["sqlalchemy.sql.operators"].Operators = object
    t = sys.modules["sqlalchemy.types"]
    t.Float, t.LargeBinary, t.TypeDecorator, t.TypeEngine, t.UserDefinedType = _Generic, _Generic, _Generic, _Generic, _Generic
    return _load("raglite._typing_ref", REF / "_typing.py")


def golden_table_rows(typing_mod: types.ModuleType) -> None:
    """What the reference's own column processors write to / read from ``chunk_embedding.embedding``
    (``_typing.py:57-78, 145-208``) for float16 embeddings as ``_embed.py:140`` produces them."""
    rng = np.random.default_rng(11)
    d, n = 24, 40
    E = rng.standard_normal((n, d)).astype(np.float32)
    E /= np.linalg.norm(E, axis=1, keepdims=True)
    E16 = E.astype(np.float16)
    # edge values a halfvec / FLOAT[] column can hold: signed zero, subnormals, the largest half, tiny and integral values
    E16[0, :8] = np.array([0.0, -0.0, 5.96e-8, -5.96e-8, 6.1e-5, 65504.0, -65504.0, 1.0], np.float16)
    E16[1, :4] = np.array([0.333251953125, 1e-3, 123.0, -0.5], np.float16)
    duck, pg, npy = typing_mod.DuckDBSingleVec(d), typing_mod.PostgresHalfVec(d), typing_mod.NumpyArray()
    duck_bind, duck_res = duck.bind_processor(None), duck.result_processor(None, None)
    pg_bind, pg_res = pg.bind_processor(None), pg.result_processor(None, None)
    lists = [duck_bind(r) for r in E16]                     # what RAGLite hands DuckDB for FLOAT[d]
    texts = [pg_bind(r) for r in E16]                       # ... and PostgreSQL for halfvec(d)
    blobs = [npy.process_bind_param(r, None) for r in E16]  # ... and any other dialect
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        from_text = np.stack([pg_res(t) for t in texts])
    from_list = np.stack([duck_res(v) for v in lists])
    from_blob = np.stack([npy.process_result_value(b, None) for b in blobs])
    counts = rng.integers(1, 5, size=64)
    row_chunk = np.repeat(np.arange(len(counts)), counts)[:n]
    np.savez_compressed(
        GOLDEN / "table_rows.npz", E16=E16, from_text=from_text, from_list=from_list, from_blob=from_blob, row_chunk=row_chunk,
        texts=np.frombuffer(json.dumps(texts).encode(), dtype=np.uint8),
        lists=np.frombuffer(json.dumps(lists).encode(), dtype=np.uint8),
        blobs=np.frombuffer(b"".join(blobs), dtype=np.uint8), blob_len=np.array([len(b) for b in blobs]))
    print("table_rows", from_text.dtype, from_list.dtype, from_blob.dtype, texts[0][:48])


def golden_rrf() -> None:
    """``reciprocal_rank_fusion`` (``_search.py:233-254``): the reference's own function text, compiled on its own
    (the module around it imports SQLAlchemy / sqlmodel), run on seeded rankings with ties and duplicates."""
    import ast
    from collections import defaultdict

    src = (REF / "_search.py").read_text()
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "reciprocal_rank_fusion")
    ns: dict = {"defaultdict": defaultdict, "ChunkId": str}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), str(REF / "_search.py"), "exec"), ns)  # noqa: S102
    rrf = ns["reciprocal_rank_fusion"]
    rng = np.random.default_rng(21)
    cases = []
    for _ in range(12):
        R, L, universe = int(rng.integers(1, 4)), int(rng.integers(1, 40)), int(rng.integers(5, 60))
        rankings = [[int(x) for x in rng.permutation(universe)[: int(rng.integers(0, L + 1))]] for _ in range(R)]
        weights = [float(w) for w in rng.choice([1.0, 0.75, 0.25, 0.5], size=R)]
        k = int(rng.choice([60, 1, 10]))
        ids, scores = rrf([[str(c) for c in r] for r in rankings], k=k, weights=weights)
        cases.append({"rankings": rankings, "weights": weights, "k": k, "ids": [int(c) for c in ids], "scores": [float(x) for x in scores]})
    # the hybrid_search call shape: two rankings, weights 0.75 / 0.25 (_search.py:271-275)
    a, b = [int(x) for x in rng.permutation(50)[:20]], [int(x) for x in rng.permutation(50)[:20]]
    ids, scores = rrf([[str(c) for c in a], [str(c) for c in b]], weights=[0.75, 0.25])
    cases.append({"rankings": [a, b], "weights": [0.75, 0.25], "k": 60, "ids": [int(c) for c in ids], "scores": [float(x) for x in scores]})
    np.savez_compressed(GOLDEN / "rrf.npz", cases=np.frombuffer(json.dumps(cases).encode(), dtype=np.uint8))
    print("rrf", len(cases), "cases")


class _FakeSaT:
    """wtpsplit-lite's ``SaT`` for the golden run: seeded float32 probabilities, one per character, a function of the
    document alone (so the fixture can store them and a test can replay them)."""

    def __init__(self, name: str) -> None:
        self.name = name

    @staticmethod
    def probas(doc: str) -> np.ndarray:
        import zlib

        rng = np.random.default_rng(zlib.crc32(doc.encode()))
        p = rng.beta(0.6, 2.0, size=len(doc))
        ends = np.array([c in ".!?。\n" for c in doc], dtype=bool)
        p[ends] = np.maximum(p[ends], rng.uniform(0.5, 1.0, size=int(ends.sum())))
        return p.astype(np.float32)

    def predict_proba(self, doc: str, **kw) -> np.ndarray:  # noqa: ANN003
        assert kw == {"stride": 128, "block_size": 256, "weighting": "hat"}, kw
        return self.probas(doc)


def golden_split_sentences() -> None:
    """``split_sentences`` (``_split_sentences.py:146-219``) and ``markdown_sentence_boundaries`` run unmodified on
    Markdown headings, whitespace runs, multi-byte text, the length edges and several (min_len, max_len) pairs, with the
    fake SaT's probabilities and with fully finite known probabilities; the infeasible case records its error."""
    for name in ("raglite", "raglite._typing", "wtpsplit_lite"):
        sys.modules.pop(name, None)
    pkg = types.ModuleType("raglite")
    pkg.__path__ = []
    sys.modules["raglite"] = pkg
    _stub("raglite._typing", FloatVector=np.ndarray)
    _stub("wtpsplit_lite", SaT=_FakeSaT)
    mod = _load("raglite._split_sentences", REF / "_split_sentences.py")
    rng = np.random.default_rng(31)
    words = "alpha beta gamma delta light clock rod frame event time of the observer velocity".split()

    def prose(n: int) -> str:
        out = []
        while sum(len(w) + 1 for w in out) < n:
            w = str(rng.choice(words))
            out.append(w + ("." if rng.random() < 0.12 else ""))
        return " ".join(out)

    docs = {
        "headings": "# Title\n\nSome text. More text here!\n\n## Section two\nBody of section. Another one.\n"
                    "### Third level\n- item one\n- item two\n#### Four\nTail text without end",
        "setext": "Heading one\n===========\n\nParagraph. Second sentence.\n\nHeading two\n-----------\nLast words here.",
        "spaces": "Alpha beta.   Gamma\tdelta.\t\tEpsilon\n\nzeta eta.\u3000\u3000Theta iota.  \n\n  Kappa.  ",
        "leading": "   \n  Leading whitespace. Then text.\t \t",
        "multibyte": "Ünïcödé tëxt — ça va? 日本語の文です。次の文。 Emoji 😀 here.\u3000Done. Ω≈ç√∫ end.",
        "len4": "abcd", "len5": "abcde", "len8": "abcdefgh", "len9": "ab cd. ef",
        "prose": prose(600),
        "long_run": "x" * 70 + " " + "y" * 150 + ". " + prose(200),
    }
    pairs = [(4, None), (4, 8), (4, 64), (4, 2048), (1, 8), (10, 2048), (3, 64)]
    cases, arrays = [], {}

    def run(name: str, doc: str, min_len: int, max_len: int | None, known: np.ndarray | None) -> None:
        i = len(cases)
        arrays[f"pred{i}"] = _FakeSaT.probas(doc)
        arrays[f"md{i}"] = mod.markdown_sentence_boundaries(doc)
        if known is not None:
            arrays[f"known{i}"] = known
        try:
            kw = {} if known is None else {"boundary_probas": known}
            out, err = mod.split_sentences(doc, min_len=min_len, max_len=max_len, **kw), None
        except ValueError as e:
            out, err = None, str(e)
        cases.append({"name": name, "doc": doc, "min_len": min_len, "max_len": max_len, "known": known is not None,
                      "sentences": out, "error": err})

    for name, doc in docs.items():
        for min_len, max_len in pairs:
            run(name, doc, min_len, max_len, None)
    for name in ("prose", "multibyte", "spaces", "long_run"):           # known probabilities override the model entirely
        doc = docs[name]
        for min_len, max_len in [(4, None), (4, 8), (4, 64), (1, 8)]:
            run(name + "_known", doc, min_len, max_len, rng.beta(0.5, 1.5, size=len(doc)))
    # no split can satisfy (5, 6) on 13 characters kept whole by stage 1 (every score is -0.25)
    run("infeasible", "abcdefghijklm", 5, 6, np.zeros(13))
    run("short13", "abcdefghijklm", 5, 6, None)
    np.savez_compressed(GOLDEN / "split_sentences.npz", cases=np.frombuffer(json.dumps(cases).encode(), dtype=np.uint8),
                        **arrays)
    print("split_sentences", len(cases), "cases,", sum(c["error"] is not None for c in cases), "errors")


def _sentences_of(doc: str) -> list[str]:
    """A document cut after every '. ', '? ', '! ' and newline (the pieces join back to the document)."""
    import re

    return [s for s in re.split(r"(?<=[.?!] )|(?<=\n)", doc) if s]


def _chunk_docs(seed: int) -> dict[str, str]:
    rng = np.random.default_rng(seed)
    words = "alpha beta gamma delta light clock rod frame event time of the observer velocity".split()

    def para(n: int) -> str:
        return " ".join(" ".join(str(w) for w in rng.choice(words, size=int(rng.integers(3, 14)))) + "."
                        for _ in range(n))

    return {
        "atx": f"# Title\n\n{para(3)}\n\n## Section\n\n{para(4)}\n\n### Deeper\n{para(2)}\n",
        "setext": f"Heading one\n===========\n\n{para(3)}\n\nHeading two\n-----------\n{para(3)}\n",
        "lists": f"{para(2)}\n\n- {para(1)}\n- {para(2)}\n- item\n\n1. first {para(1)}\n2. second\n\n{para(2)}\n",
        "quotes": f"{para(2)}\n\n> {para(2)}\n> {para(1)}\n\n{para(3)}\n",
        "consecutive": f"# A\n## B\n### C\n- x\n- y\n> q\n\n{para(2)}\n# D\n\n{para(5)}\n",
        "whitespace": f"{para(2)}\n\n   \n\t\n\n{para(3)}\n  \n",
        "prose": para(40),
    }


def golden_split_chunklets() -> None:
    """``split_chunklets`` and ``markdown_chunklet_boundaries`` (``_split_chunklets.py``) run unmodified on Markdown
    headings (ATX and setext), lists, block quotes, consecutive boundaries, whitespace-only sentences, a sentence longer
    than max_size and one sentence, at several max_size values; the empty document records its error."""
    for name in ("raglite", "raglite._typing"):
        sys.modules.pop(name, None)
    pkg = types.ModuleType("raglite")
    pkg.__path__ = []
    sys.modules["raglite"] = pkg
    _stub("raglite._typing", FloatVector=np.ndarray)
    mod = _load("raglite._split_chunklets", REF / "_split_chunklets.py")
    docs = {k: _sentences_of(v) for k, v in _chunk_docs(41).items()}
    docs["long_middle"] = ["a b. "] * 5 + ["x" * 50] + ["c d. "] * 5
    docs["long_first"] = ["x" * 50] + ["a b. "] * 5 + ["c d. "] * 5
    docs["long_first_short"] = ["x" * 50] + ["c d. "] * 5
    docs["one"] = ["Just one sentence."]
    docs["spaces_only"] = ["   ", "\n", " \t "]
    cases = []
    for name, sents in docs.items():
        for max_size in (20, 64, 256, 2048):
            out = mod.split_chunklets(sents, max_size=max_size)
            cases.append({"name": name, "sentences": sents, "max_size": max_size, "chunklets": out, "error": None,
                          "md": mod.markdown_chunklet_boundaries(sents).tolist(),
                          "statements": mod.compute_num_statements(sents).tolist()})
    try:
        mod.split_chunklets([])
    except ValueError as e:
        cases.append({"name": "empty", "sentences": [], "max_size": 2048, "chunklets": None, "error": str(e)})
    np.savez_compressed(GOLDEN / "split_chunklets.npz", cases=np.frombuffer(json.dumps(cases).encode(), dtype=np.uint8))
    print("split_chunklets", len(cases), "cases")


def golden_split_chunks() -> None:
    """``split_chunks`` (``_split_chunks.py``) run unmodified on seeded fp16 and fp32 chunklet embeddings: Markdown
    headings, several max_size values, identical rows (the projection is skipped), and the long-chunklet and zero-norm
    errors.  Each solved case also stores the float32 cost vector the reference hands to ``linprog``."""
    for name in ("raglite", "raglite._typing"):
        sys.modules.pop(name, None)
    pkg = types.ModuleType("raglite")
    pkg.__path__ = []
    sys.modules["raglite"] = pkg
    _stub("raglite._typing", FloatMatrix=np.ndarray)
    mod = _load("raglite._split_chunks", REF / "_split_chunks.py")
    seen: list[np.ndarray] = []
    real_linprog = mod.linprog

    def spy(c, **kw):  # noqa: ANN001, ANN003, ANN202
        seen.append(np.array(c, copy=True))
        return real_linprog(c, **kw)

    mod.linprog = spy
    rng = np.random.default_rng(43)
    cases, arrays = [], {}

    def run(name: str, chunklets: list[str], emb: np.ndarray, max_size: int) -> None:
        i = len(cases)
        arrays[f"emb{i}"] = emb
        seen.clear()
        try:
            chunks, _ = mod.split_chunks(chunklets, emb, max_size=max_size)
            err = None
        except ValueError as e:
            chunks, err = None, str(e)
        if seen:
            arrays[f"cost{i}"] = seen[0]
        cases.append({"name": name, "chunklets": chunklets, "max_size": max_size, "chunks": chunks, "error": err,
                      "solved": bool(seen)})

    def rows(n: int, d: int, dtype: type, topics: int = 4) -> np.ndarray:
        centers = rng.standard_normal((topics, d))
        which = np.sort(rng.integers(0, topics, size=n))
        return (centers[which] + 0.8 * rng.standard_normal((n, d))).astype(dtype)

    words = "alpha beta gamma delta light clock rod frame event time of the observer velocity".split()
    for k in range(24):
        n = int(rng.integers(3, 80))
        chunklets = []
        for _ in range(n):
            body = " ".join(str(w) for w in rng.choice(words, size=int(rng.integers(3, 90)))) + ". "
            chunklets.append(("# " + body[:30] + "\n") if rng.random() < 0.2 else body)
        emb = rows(n, int(rng.choice([16, 48, 64])), np.float16 if k % 3 else np.float32)
        for max_size in (600, 2048):
            run(f"doc{k}", chunklets, emb, max_size)
    same = ["alpha beta gamma. " * 3] * 12
    run("identical_rows", same, np.tile(rng.standard_normal((1, 32)).astype(np.float16), (12, 1)), 128)
    run("identical_rows_f32", same, np.tile(rng.standard_normal((1, 32)).astype(np.float32), (12, 1)), 200)
    run("one_chunklet", ["# Only\n"], rows(1, 16, np.float16), 64)
    run("fits", ["a. ", "b. ", "c. "], rows(3, 16, np.float16), 64)
    run("too_long", ["a" * 70, "b. "], rows(2, 16, np.float16), 64)
    zero = rows(4, 16, np.float16)
    zero[2] = 0
    run("zero_norm", ["a. " * 10, "b. " * 10, "c. " * 10, "d. " * 10], zero, 40)
    np.savez_compressed(GOLDEN / "split_chunks.npz", cases=np.frombuffer(json.dumps(cases).encode(), dtype=np.uint8),
                        **arrays)
    print("split_chunks", len(cases), "cases,", sum(c["solved"] for c in cases), "solved")


def golden_chatml_tools() -> None:
    """The function-calling chat handler: its template rendered with jinja2 as the handler renders it, and the handler
    run over a scripted Llama (each completion returns a given raw output cut at its first stop string, as
    llama-cpp-python's create_completion does), recording every completion's prompt, grammar and settings."""
    import ast

    import jinja2
    from jinja2.sandbox import ImmutableSandboxedEnvironment

    src = (REF / "_chatml_function_calling.py").read_text()
    tree = ast.parse(src)
    tmpl = next(ast.literal_eval(n.value) for n in ast.walk(tree) if isinstance(n, ast.Assign)
                and any(getattr(t, "id", "") == "function_calling_template" for t in n.targets))
    render = ImmutableSandboxedEnvironment(undefined=jinja2.StrictUndefined).from_string(tmpl).render

    def tool(name: str, desc: str | None, props: dict) -> dict:
        f = {"name": name, "parameters": {"type": "object", "properties": props, "required": list(props),
                                          "additionalProperties": False}}
        if desc is not None:
            f["description"] = desc
        return {"type": "function", "function": f}

    kb = tool("search_knowledge_base", "Search the knowledge base.\nIMPORTANT: You MAY NOT use this function if the "
              "question can be answered with common knowledge or straightforward reasoning.\nFor multi-faceted "
              "questions, call this function once for each facet.",
              {"query": {"type": "string", "description": "The `query` string MUST be a precise single-faceted question "
                         "in the user's language.\nThe `query` string MUST resolve all pronouns to explicit nouns."}})
    odd = tool("lookup", '  Quotes "q", \'s\', <tag> & amp; café  ', {"k": {"type": "integer", "description": "a<b"}})
    plain = tool("plain", None, {"x": {"type": "string", "maxLength": 8}})
    call = {"role": "assistant", "content": None, "tool_calls": [
        {"id": "call__0_search_knowledge_base_x", "type": "function",
         "function": {"name": "search_knowledge_base", "arguments": '{"query": "What is a fox?"}'}},
        {"id": "call__1_search_knowledge_base_x", "type": "function",
         "function": {"name": "search_knowledge_base", "arguments": '{"query": "dogs"}'}}]}
    toolmsg = {"role": "tool", "content": '{"documents": [{"id": "d"}]}', "tool_call_id": "call__0_x"}
    lists = {
        "user": [{"role": "user", "content": "What colour is the fox?"}],
        "user_sys_appended": [{"role": "user", "content": "Hi & <b>"}, {"role": "system", "content": ""}],
        "system_user": [{"role": "system", "content": "Be brief."}, {"role": "user", "content": "Tell me 'this'."}],
        "history": [{"role": "system", "content": "S"}, {"role": "user", "content": "q1"},
                    {"role": "assistant", "content": "a1"}, {"role": "user", "content": "q2"}],
        "tool_round": [{"role": "user", "content": "What colour is the fox?"}, call, toolmsg,
                       {**toolmsg, "tool_call_id": "call__1_x"}],
        "tool_round_answered": [{"role": "user", "content": "Q"}, call, toolmsg, {"role": "assistant", "content": "A."}],
    }
    toolsets = {"kb": [kb], "odd": [odd, kb], "plain": [plain]}
    renders = []
    for ln, msgs in lists.items():
        renders.append({"messages": ln, "tools": None, "tool_calls": False,
                        "text": render(messages=msgs, tools=[], tool_calls=None, add_generation_prompt=True)})
        for tn, tools in toolsets.items():
            renders.append({"messages": ln, "tools": tn, "tool_calls": True,
                            "text": render(messages=msgs, tools=tools, tool_calls=True, add_generation_prompt=True)})

    class Grammar:
        def __init__(self, kind: str, text: str) -> None:
            self.kind, self.text = kind, text

    class LlamaGrammar:
        @staticmethod
        def from_string(text: str, verbose: bool = False) -> Grammar:  # noqa: ARG004
            return Grammar("gbnf", text)

        @staticmethod
        def from_json_schema(text: str, verbose: bool = False) -> Grammar:  # noqa: ARG004
            return Grammar("json_schema", text)

    class ScriptedLlama:
        verbose = False

        def __init__(self, raw: list[str]) -> None:
            self.raw, self.calls = list(raw), []

        def create_completion(self, prompt: str, **kw):  # noqa: ANN003, ANN202
            raw = self.raw.pop(0)
            stops = kw.get("stop") or []
            cut = min([i for i in (raw.find(x) for x in stops) if i >= 0], default=len(raw))
            g = kw.get("grammar")
            self.calls.append({"prompt": prompt, "grammar": None if g is None else [g.kind, g.text],
                               "temperature": kw["temperature"], "stop": list(stops), "max_tokens": kw["max_tokens"]})
            return {"id": "cmpl-x", "created": 0, "model": "m",
                    "choices": [{"text": raw[:cut], "index": 0, "logprobs": None, "finish_reason": "stop"}]}

    class _Lazy(types.ModuleType):
        def __getattr__(self, name):  # noqa: ANN001, ANN204
            return type(name, (), {})

    lazy = _Lazy("raglite._lazy_llama")
    lazy.llama = _Lazy("llama")
    lazy.llama_types = _Lazy("llama_types")
    lazy.llama_grammar = types.SimpleNamespace(LlamaGrammar=LlamaGrammar)
    lazy.llama_chat_format = types.SimpleNamespace(_convert_completion_to_chat=lambda c, stream=False: c)  # noqa: ARG005
    sys.modules.setdefault("raglite", types.ModuleType("raglite"))
    sys.modules["raglite._lazy_llama"] = lazy
    handler = _load("raglite._chatml_function_calling_ref", REF / "_chatml_function_calling.py")

    fn = "functions.search_knowledge_base:"
    args = ['{"query": "What colour is the fox?"}', '{ "query":"dogs" }\n ', '{"query": "caf\\u00e9 <&>"}']
    end = "<|im_end|>"
    scenarios = {
        "message": ("auto", "kb", ["<message>", "The fox is brown." + end]),
        "think_message": ("auto", "kb", ["<think>\nmaybe not</think>\n\n<message>", "Brown." + end]),
        "one_call": ("auto", "kb", ["<function_calls>\n" + fn, args[0] + end, "</function_calls>"]),
        "two_calls": ("auto", "kb", ["<function_calls>\n" + fn, args[0] + end, fn, args[1] + end, end]),
        "think_call": ("auto", "kb", ["<think>\nsearch</think>\n\n<function_calls>\n" + fn, args[2] + end,
                                      "</function_calls>"]),
        "cap": ("auto", "kb", ["<function_calls>\n" + fn] + [x for i in range(17) for x in (
            '{"query": "q%d"}' % i + end, fn)]),
        "unknown_name": ("auto", "odd", ["<function_calls>\nfunctions.lookup:", '{"k": 3}' + end, end]),
        "fixed": ({"type": "function", "function": {"name": "plain"}}, "plain",
                  ["<function_calls>\nfunctions.plain:", '{"x": "abc"}' + end, "<|endoftext|>"]),
    }
    protocol = []
    for name, (choice, tn, raw) in scenarios.items():
        for ln in ("user",) if name == "cap" else ("user", "system_user"):
            llm = ScriptedLlama(raw)
            out = handler.chatml_function_calling_with_streaming(llm, [dict(m) for m in lists[ln]],
                                                                 tools=toolsets[tn], tool_choice=choice,
                                                                 temperature=0.6, top_p=0.95, top_k=20, min_p=0.0)
            msg = out["choices"][0].get("message")
            result = ({"tool_calls": [[c["function"]["name"], c["function"]["arguments"]] for c in msg["tool_calls"]]}
                      if msg else {"text": out["choices"][0]["text"]})
            protocol.append({"scenario": name, "messages": ln, "tools": tn, "tool_choice": choice, "raw": raw,
                             "calls": llm.calls, "result": result, "unused_raw": len(llm.raw)})
    data = {"lists": lists, "toolsets": toolsets, "renders": renders, "protocol": protocol}
    (GOLDEN / "chatml_tools.json").write_text(json.dumps(data, ensure_ascii=False) + "\n")
    print("chatml_tools", len(renders), "renders,", len(protocol), "protocol runs")


if __name__ == "__main__":
    GOLDEN.mkdir(parents=True, exist_ok=True)
    golden_rrf()
    embed_mod, qa_mod = install_reference_stubs()
    golden_pool(embed_mod)
    golden_adapter(qa_mod)
    golden_table_rows(load_reference_typing())
    golden_split_sentences()
    golden_split_chunklets()
    golden_split_chunks()
    golden_chatml_tools()

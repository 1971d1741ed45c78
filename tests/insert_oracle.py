"""Host oracle of ingest: RAGLite's document and chunk records (``_database.py:51-277``, ``_insert.py:102-111``) restated
in plain Python, the ``standard`` embedding type's blend as the literal NumPy float16 expression (``_insert.py:141``)
and as an explicit float32-then-round statement, and the metadata containment ``delete_documents_by_metadata``
selects with (``_delete.py:48-64``)."""

from __future__ import annotations

import hashlib
from typing import Any

import numpy as np
from markdown_it import MarkdownIt

from raglite_b200 import Chunk

ALPHA = 0.15


def listify(metadata: dict[str, Any] | None) -> dict[str, list[Any]]:
    out = {}
    for k, v in (metadata or {}).items():
        out[k] = v if isinstance(v, list) else [v]
    return out


def sha16(text: str) -> str:
    return hashlib.sha256(text.encode()).hexdigest()[:16]


def document_fields(content: str, *, id: str | None = None, url: str | None = None,  # noqa: A002
                    filename: str | None = None, **kwargs: Any) -> dict[str, Any]:
    """``Document.from_text``'s fields."""
    line = content.strip().split("\n", 1)[0].strip()
    if len(line) > 80:  # noqa: PLR2004
        line = line[:80] + "..."
    meta = {"filename": filename or line, "uri": id, "url": url, "size": len(content.encode())}
    meta.update(kwargs)
    return {"id": sha16(content) if id is None else id, "filename": filename or line, "url": url,
            "metadata_": listify(meta), "content": content}


def heading_lines(doc: str, leading_only: bool = False) -> list[str]:  # noqa: FBT001, FBT002
    lines = ["", "", "", "", "", ""]
    level = None
    for token in MarkdownIt().parse(doc):
        if token.type == "heading_open":
            level = int(token.tag[1])
            continue
        if token.type == "heading_close":
            level = None
            continue
        if level is not None:
            lines[level - 1] = "#" * level + " " + token.content.strip().replace("\n", " ")
            for j in range(level, 6):
                lines[j] = ""
        elif leading_only and token.content and not token.content.isspace():
            break
    return lines


def truncated(headings: str, body: str) -> str:
    lines = heading_lines(headings)
    leading = heading_lines(body, leading_only=True)
    for i, line in enumerate(leading):
        if line:
            for j in range(i, 6):
                lines[j] = ""
            break
    return "\n".join(h for h in lines if h)


def records(doc_id: str, filename: str, url: str | None, metadata: dict[str, Any], bodies: list[str]) -> list[Chunk]:
    """The chunk records ``_create_chunk_records`` makes of a document's chunks."""
    out = []
    carried = ""
    for i, body in enumerate(bodies):
        meta = {"filename": filename, "url": url}
        meta.update(metadata)
        c = Chunk(id=sha16(f"{doc_id}-{i}"), document_id=doc_id, index=i, headings=truncated(carried, body), body=body,
                  metadata_=listify(meta))
        out.append(c)
        carried = "\n".join(h for h in heading_lines(c.headings + "\n\n" + c.body) if h)
    return out


def blend_numpy(e: np.ndarray, f: np.ndarray) -> np.ndarray:
    """The reference's expression on float16 rows, literally."""
    α = ALPHA  # noqa: PLC2401
    with np.errstate(over="ignore", invalid="ignore"):
        return α * e + (1 - α) * f


def blend_f32(e: np.ndarray, f: np.ndarray) -> np.ndarray:
    """Each weight rounded to float16; each product and the sum computed in float32 and rounded to float16."""
    a = np.float32(np.float16(ALPHA))
    b = np.float32(np.float16(1 - ALPHA))
    with np.errstate(over="ignore", invalid="ignore"):
        p = (a * np.asarray(e, np.float16).astype(np.float32)).astype(np.float16)
        q = (b * np.asarray(f, np.float16).astype(np.float32)).astype(np.float16)
        return (p.astype(np.float32) + q.astype(np.float32)).astype(np.float16)


def contains(metadata: dict[str, Any], metadata_filter: dict[str, Any]) -> bool:
    """JSON containment of the listified filter in list-valued metadata."""
    for k, vs in listify(metadata_filter).items():
        have = metadata.get(k)
        if have is None and k not in metadata:
            return False
        have = have if isinstance(have, list) else [have]
        if any(v not in have for v in vs):
            return False
    return True

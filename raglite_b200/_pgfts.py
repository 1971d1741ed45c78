"""PostgreSQL full-text search as the reference's PostgreSQL ``keyword_search`` uses it (``_search.py:176-201``):
``ts_rank(to_tsvector('simple', body), to_tsquery('simple', tsv_query))`` with ``tsv_query`` the query's words joined by
``" | "`` once ASCII punctuation is replaced by spaces.

Document side: the index takes the database's own ``to_tsvector('simple', body)::text`` (``parse_tsvector``) rather than
restating PostgreSQL's 23-token-type parser.  Query side: after the punctuation strip an operand holds no ASCII
punctuation and no whitespace, so the parser and the ``simple`` dictionary reduce to the few rules of ``query_lexemes``.

What is restated here is recalled from PostgreSQL's sources (``to_tsany.c``, ``ts_parse.c``, ``tsvector.c``,
``tsrank.c``), not checked against a server (DESIGN.md section 5).  Input those rules do not cover is refused, not guessed.
"""

from __future__ import annotations

import re
import string
from typing import Any

MAX_POSITIONS = 256      # MAXNUMPOS: positions a tsvector keeps per lexeme
MAX_POSITION = 16383     # MAXENTRYPOS - 1: larger positions are stored as this
MAX_TOKEN_BYTES = 2047   # MAXSTRLEN: a token of this many UTF-8 bytes or more is not indexed

TSVECTOR_SELECT = "SELECT id, to_tsvector('simple', body)::text FROM chunk"

_PUNCT_TO_SPACE = str.maketrans(dict.fromkeys(string.punctuation, " "))


def tsquery_operands(query: str) -> list[str]:
    """The operands the reference joins with ``" | "``: every ASCII punctuation character becomes a space, then
    ``str.split()`` (any Unicode whitespace)."""
    return query.translate(_PUNCT_TO_SPACE).split()


def _lower(c: str) -> str:
    """glibc ``towlower`` of one character: Python's lower case where it is one character, no context rules (so ``Σ`` is
    always ``σ``), and ``İ`` (U+0130) -> ``i``."""
    low = c.lower()
    if len(low) == 1:
        return low
    return "i" if c == "İ" else c


def _pieces(operand: str) -> list[str]:
    """The tokens of the default parser within one operand: runs of letters (``str.isalpha``) and ASCII digits."""
    out, run = [], []
    for c in operand:
        if c.isalpha() or "0" <= c <= "9":
            run.append(c)
        elif run:
            out.append("".join(run))
            run = []
    if run:
        out.append("".join(run))
    return out


def operand_lexeme(operand: str) -> str | None:
    """The lexeme ``to_tsquery('simple', ...)`` makes of one operand, or ``None`` when the operand is dropped (no token,
    or a token of ``MAX_TOKEN_BYTES`` bytes or more).  An operand of two or more tokens becomes a phrase (``'a' <-> 'b'``),
    whose matching needs positions: ``NotImplementedError``."""
    pieces = _pieces(operand)
    if len(pieces) > 1:
        raise NotImplementedError(f"the query operand {operand!r} is a phrase for PostgreSQL ({' <-> '.join(pieces)}): "
                                  "ts_rank of phrase operands needs positions and is not implemented")
    if not pieces or len(pieces[0].encode()) >= MAX_TOKEN_BYTES:
        return None
    return "".join(_lower(c) for c in pieces[0])


def query_lexemes(query: str) -> list[str]:
    """The entries of the query's ``tsquery``: its distinct lexemes in ascending UTF-8 byte order (``SortAndUniqItems``).
    Empty: the query matches nothing (``@@`` with an empty ``tsquery`` is false)."""
    lex = {x for x in (operand_lexeme(op) for op in tsquery_operands(query)) if x is not None}
    return sorted(lex, key=lambda s: s.encode())


_ENTRY = re.compile(r"'((?:[^'\\]|''|\\\\)*)'(?::([^ ]*))?")
_POS = r"(?:[1-9][0-9]{0,3}|1[0-5][0-9]{3}|16[0-2][0-9]{2}|163[0-7][0-9]|1638[0-3])"   # 1..16383
_POSITIONS = re.compile(rf"{_POS}(?:,{_POS})*")


def parse_tsvector(text: Any, chunk_id: Any = None) -> tuple[list[str], list[int]]:
    """``(lexemes, npos)`` of one ``tsvector`` in PostgreSQL's text output: space-separated ``'lexeme'`` entries (``'`` and
    ``\\`` doubled inside the quotes), each with an optional ``:p1,p2,...`` list of positions in 1..16383.  ``npos`` is the
    number of positions listed; a lexeme without positions (a stripped tsvector) counts as one.  Weight letters
    ``A``/``B``/``C``, more than 256 positions, a position outside 1..16383, a repeated lexeme, and anything else that
    ``to_tsvector(...)::text`` does not print raise ``ValueError`` naming ``chunk_id``.  Only the number of positions is
    kept, so their order is not checked."""
    def bad(why: str) -> ValueError:
        return ValueError(f"tsvector of chunk {chunk_id!r}: {why}")

    if not isinstance(text, str):
        raise bad(f"expected the text of to_tsvector(...)::text, got {type(text).__name__}")
    lexemes: list[str] = []
    npos: list[int] = []
    pos, n = 0, len(text)
    while pos < n:
        m = _ENTRY.match(text, pos)
        if m is None:
            raise bad(f"malformed entry at character {pos}: {text[pos:pos + 40]!r}")
        lex = m.group(1).replace("''", "'").replace("\\\\", "\\")
        if not lex:
            raise bad("empty lexeme")
        ps = m.group(2)
        if ps is None:
            count = 1
        else:
            if any(w in ps for w in "ABC"):
                raise bad(f"lexeme {lex!r} has weighted positions ({ps}); only weight D (to_tsvector's) is ranked")
            if _POSITIONS.fullmatch(ps) is None:
                raise bad(f"positions {ps!r} of lexeme {lex!r} are not a list of integers in 1..{MAX_POSITION}")
            count = ps.count(",") + 1
            if count > MAX_POSITIONS:
                raise bad(f"lexeme {lex!r} lists {count} positions; a tsvector keeps at most {MAX_POSITIONS}")
        lexemes.append(lex)
        npos.append(count)
        pos = m.end()
        if pos < n:
            if text[pos] != " " or pos + 1 == n:
                raise bad(f"malformed separator at character {pos}")
            pos += 1
    if len(set(lexemes)) != len(lexemes):
        raise bad("a lexeme is listed twice")
    return lexemes, npos

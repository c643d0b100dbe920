"""Long inputs: the text of a request cut into segments, each spoken as its own row (DESIGN.md, "Long inputs").

``split_text(text, max_chars)`` follows one deterministic rule:

1. Sentences.  The text is cut after every run of sentence-final marks -- ``. ! ? ;`` when followed by whitespace or the
   end of the text, the CJK ``。！？；`` anywhere -- and after every newline.
2. Whitespace at each cut is dropped: every piece is stripped, and pieces that are empty (blank lines, trailing
   whitespace) are dropped.
3. Hard cuts.  A piece longer than ``max_chars`` is cut after the last whitespace or punctuation mark (``, : 、 ， ：``
   and the marks above) among its first ``max_chars`` characters, or after ``max_chars`` characters when there is none;
   the rest is cut again the same way.
4. Merges.  A piece shorter than ``min_chars`` (default ``min(MIN_CHARS, max_chars)``) is merged with the next piece,
   the text between them included, while the result is at most ``max_chars`` long.

So every segment is 1 .. ``max_chars`` characters of the input, in order, and the input is the segments joined with the
whitespace that was dropped at the cuts.  A text of whitespace alone has no segment.

Seeds.  Segment k of a request with seed ``s`` draws its uniforms from ``take_uniforms(segment_seed(s, k), n)`` (model.py),
``segment_seed(s, k) = (s + k * 0x9E3779B97F4A7C15) mod 2^63``: segment k alone, spoken with those uniforms, gives the
same codes.
"""
from __future__ import annotations

from typing import List, Tuple

MIN_CHARS = 24
MAX_CHARS = 400                 # default of ``max_segment_chars``
CHARS_PER_S = 14.0              # speech the scheduler expects from text not yet spoken (serving.py)
_ASCII_END = ".!?;"
_CJK_END = "。！？；"
_SOFT = ",:、，：" + _ASCII_END + _CJK_END


def check_max_chars(max_chars) -> int:
    if isinstance(max_chars, bool) or not isinstance(max_chars, int) or max_chars < 1:
        raise ValueError(f"max_segment_chars must be a positive integer, got {max_chars!r}")
    return max_chars


def _sentences(text: str) -> List[Tuple[int, int]]:
    spans, start, n = [], 0, len(text)
    for i, c in enumerate(text):
        nxt = text[i + 1] if i + 1 < n else ""
        cut = c == "\n"
        if c in _CJK_END and nxt not in _CJK_END:
            cut = True
        if c in _ASCII_END and (nxt == "" or nxt.isspace()):
            cut = True
        if cut:
            spans.append((start, i + 1))
            start = i + 1
    if start < n:
        spans.append((start, n))
    return spans


def _strip(text: str, a: int, b: int) -> Tuple[int, int]:
    while a < b and text[a].isspace():
        a += 1
    while b > a and text[b - 1].isspace():
        b -= 1
    return a, b


def _hard_cut(text: str, a: int, b: int, max_chars: int) -> List[Tuple[int, int]]:
    out = []
    while b - a > max_chars:
        cut = a + max_chars
        for i in range(a + max_chars - 1, a, -1):
            if text[i].isspace() or text[i] in _SOFT:
                cut = i + 1
                break
        p = _strip(text, a, cut)
        if p[0] < p[1]:
            out.append(p)
        a = _strip(text, cut, b)[0]
    if a < b:
        out.append((a, b))
    return out


def split_spans(text: str, max_chars: int = MAX_CHARS, min_chars=None) -> List[Tuple[int, int]]:
    """the segments of ``text`` as (start, end) character spans (module docstring)"""
    max_chars = check_max_chars(max_chars)
    min_chars = min(MIN_CHARS, max_chars) if min_chars is None else int(min_chars)
    pieces = []
    for a, b in _sentences(text):
        a, b = _strip(text, a, b)
        if a < b:
            pieces.extend(_hard_cut(text, a, b, max_chars))
    merged: List[Tuple[int, int]] = []
    for a, b in pieces:
        if merged and merged[-1][1] - merged[-1][0] < min_chars and b - merged[-1][0] <= max_chars:
            merged[-1] = (merged[-1][0], b)
        else:
            merged.append((a, b))
    return merged


def split_text(text: str, max_chars: int = MAX_CHARS, min_chars=None) -> List[str]:
    """``text`` cut into segments of at most ``max_chars`` characters by the rule of the module docstring"""
    return [text[a:b] for a, b in split_spans(text, max_chars, min_chars)]


def segment_seed(seed: int, k: int) -> int:
    """the seed of segment k of a request with seed ``seed`` (module docstring)"""
    return (int(seed) + int(k) * 0x9E3779B97F4A7C15) % (1 << 63)

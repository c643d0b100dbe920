"""SSML input: a subset of the Speech Synthesis Markup Language, spoken as segment rows (DESIGN.md, "SSML").

A document is parsed with the standard library's expat parser.  It comes from outside the program, so a DOCTYPE, an
entity declaration or a processing instruction is refused before anything else is read.

Elements and attributes (anything else -- ``mark``, ``say-as``, ``emphasis``, ``phoneme``, ``audio``, ``lang``, vendor
tags such as ``amazon:effect`` -- and any other attribute is refused, with the element or attribute and its line and
column in the message; so are malformed XML and a document with no text to speak):

* ``<speak>`` is the required root, with ``version``, ``xmlns`` and ``xml:lang``.
* ``<p>`` and ``<s>`` force a cut at both edges; they take ``xml:lang``.
* ``<break time="..." strength="..."/>``: ``time`` is ``N ms`` or ``N s`` (decimals allowed, rounded to whole ms) and
  wins over ``strength``; ``strength`` is none 0, x-weak 250, weak 500, medium 750, strong 1000, x-strong 1250 ms; a
  break with neither is medium.  A break is a cut.  Breaks with nothing but whitespace between them add up, and one
  boundary holds at most ``join.BREAK_MAX_MS`` (10 000 ms).
* ``<prosody rate pitch volume>``; nested values compose: rates multiply, semitones add, dB add.
  ``rate``: ``N%`` is the factor N/100, ``+N%`` / ``-N%`` the factor 1 +- N/100, a bare positive number is a factor,
  x-slow 0.5, slow 0.75, medium 1, fast 1.25, x-fast 1.75.  ``pitch``: ``[+-]Nst``; ``+N%`` / ``-N%`` is
  12 log2(1 +- N/100) semitones; x-low -6, low -3, medium 0, high +3, x-high +6.  ``volume``: ``[+-]NdB``; silent -96,
  x-soft -12, soft -6, medium 0, loud +6, x-loud +12.  Hz forms, ``contour``, ``range`` and ``duration`` are refused.
  The composed values of every span that holds text must pass ``resample.check_prosody`` (the tempo's q range
  included); the error names the span.
* ``<voice name="...">``: ``name`` is looked up in the caller's ``voices`` mapping (the innermost voice wins); an
  unknown name is refused with the known ones.  Text outside every ``<voice>`` is spoken by the call's default voice.
* ``<sub alias="...">`` is spoken as ``alias``; its content must be text only.

Text.  Every run of whitespace, newlines included, becomes one space.  A maximal run of text with one voice, one
prosody and one language and no cut inside it is cut into segments by the unchanged ``segment.split_text(run,
max_segment_chars)``; so ``<speak>T</speak>`` with T on one line gives exactly ``split_text(T)``.

Language.  The innermost ``xml:lang``, mapped by its primary subtag (zh, en, ja, ko, de, fr, ru, pt, es, it; any other
is refused); without one, the voice spec's ``"language"``; without that, the call's ``language``.

Pauses.  ``breaks`` has one entry per boundary, S + 1 for S segments: entry 0 is before the first segment (leading
silence), entry S after the last (trailing silence), entry k between segments k - 1 and k.  It is the sum of the breaks
at that boundary, or None where the document has none: the request's ``pause_ms`` then applies (0 at the two outer
boundaries).  A break adds to the silence the model itself makes at a segment's edges, as ``pause_ms`` does.

Seeds.  Segment k of a document uses ``segment.segment_seed(seed, k)``, as ``split=True`` does.
"""
from __future__ import annotations

import math
import re
import xml.parsers.expat
from dataclasses import dataclass
from typing import List, Mapping, Optional

STRENGTH_MS = {"none": 0, "x-weak": 250, "weak": 500, "medium": 750, "strong": 1000, "x-strong": 1250}
RATES = {"x-slow": 0.5, "slow": 0.75, "medium": 1.0, "fast": 1.25, "x-fast": 1.75}
PITCHES = {"x-low": -6.0, "low": -3.0, "medium": 0.0, "high": 3.0, "x-high": 6.0}
VOLUMES = {"silent": -96.0, "x-soft": -12.0, "soft": -6.0, "medium": 0.0, "loud": 6.0, "x-loud": 12.0}
LANGUAGES = {"zh": "Chinese", "en": "English", "ja": "Japanese", "ko": "Korean", "de": "German", "fr": "French",
             "ru": "Russian", "pt": "Portuguese", "es": "Spanish", "it": "Italian"}
ATTRIBUTES = {"speak": {"version", "xmlns", "xml:lang"}, "p": {"xml:lang"}, "s": {"xml:lang"},
              "break": {"time", "strength"}, "prosody": {"rate", "pitch", "volume"}, "voice": {"name"},
              "sub": {"alias"}}
_NUM = r"(\d+(?:\.\d*)?|\.\d+)"


@dataclass(frozen=True)
class Span:
    """one segment of a document: its text, the name of its voice, its language and its prosody"""
    text: str
    voice: Optional[str]
    language: str
    speed: float = 1.0
    pitch: float = 0.0
    gain_db: float = 0.0


@dataclass
class Document:
    spans: List[Span]
    breaks: List[Optional[int]]    # S + 1 boundaries, ms; None where the document has no break


class _Node:
    def __init__(self, tag, attrs, where):
        self.tag, self.attrs, self.where, self.children = tag, attrs, where, []


def _parse_xml(ssml: str) -> _Node:
    if not isinstance(ssml, str):
        raise ValueError(f"an SSML document is a string, got {type(ssml).__name__}")
    p = xml.parsers.expat.ParserCreate()
    p.SetParamEntityParsing(xml.parsers.expat.XML_PARAM_ENTITY_PARSING_NEVER)
    stack: List[_Node] = []
    root: List[_Node] = []

    def where():
        return f"line {p.CurrentLineNumber}, column {p.CurrentColumnNumber + 1}"

    def refuse(what):
        def handler(*_):
            raise ValueError(f"SSML: {what} is not accepted ({where()})")
        return handler

    def start(tag, attrs):
        node = _Node(tag, attrs, where())
        (stack[-1].children if stack else root).append(node)
        stack.append(node)

    def end(tag):
        stack.pop()

    def text(data):
        if stack:
            stack[-1].children.append(data)

    p.StartDoctypeDeclHandler = refuse("a DOCTYPE")
    p.EntityDeclHandler = refuse("an entity declaration")
    p.UnparsedEntityDeclHandler = refuse("an entity declaration")
    p.ExternalEntityRefHandler = refuse("an external entity")
    p.ProcessingInstructionHandler = refuse("a processing instruction")
    p.StartElementHandler, p.EndElementHandler, p.CharacterDataHandler = start, end, text
    try:
        p.Parse(ssml, True)
    except xml.parsers.expat.ExpatError as ex:
        raise ValueError(f"SSML: malformed XML: {ex}") from None
    if root[0].tag != "speak":
        raise ValueError(f"SSML: the root element must be <speak>, got <{root[0].tag}> ({root[0].where})")
    return root[0]


def _bad(node: _Node, name: str, value: str, why: str = "") -> ValueError:
    return ValueError(f"SSML: <{node.tag}> {name}={value!r} is not accepted{': ' + why if why else ''} ({node.where})")


def break_ms(node: _Node) -> int:
    """the silence of one ``<break>``, in whole ms"""
    time, strength = node.attrs.get("time"), node.attrs.get("strength")
    if time is not None:
        m = re.fullmatch(_NUM + r"\s*(ms|s)", time.strip())
        if not m:
            raise _bad(node, "time", time, "use N ms or N s")
        v = float(m.group(1)) * (1 if m.group(2) == "ms" else 1000)
        return int(math.floor(v + 0.5))
    if strength is not None:
        if strength not in STRENGTH_MS:
            raise _bad(node, "strength", strength, f"use one of {', '.join(STRENGTH_MS)}")
        return STRENGTH_MS[strength]
    return STRENGTH_MS["medium"]


def rate_factor(node: _Node, value: str) -> float:
    v = value.strip()
    if v in RATES:
        return RATES[v]
    m = re.fullmatch(r"([+-]?)" + _NUM + "%", v)
    if m:
        x = float(m.group(2)) / 100
        return {"": x, "+": 1 + x, "-": 1 - x}[m.group(1)]
    m = re.fullmatch(_NUM, v)
    if m and float(m.group(1)) > 0:
        return float(m.group(1))
    raise _bad(node, "rate", value, "use N%, +N%, -N%, a positive number or x-slow .. x-fast")


def pitch_semitones(node: _Node, value: str) -> float:
    v = value.strip()
    if v in PITCHES:
        return PITCHES[v]
    m = re.fullmatch(r"([+-]?)" + _NUM + "st", v)
    if m:
        return float(m.group(1) + m.group(2))
    m = re.fullmatch(r"([+-])" + _NUM + "%", v)
    if m:
        x = 1 + float(m.group(1) + m.group(2)) / 100
        if x > 0:
            return 12 * math.log2(x)
    raise _bad(node, "pitch", value, "use +-Nst, +-N% or x-low .. x-high")


def volume_db(node: _Node, value: str) -> float:
    v = value.strip()
    if v in VOLUMES:
        return VOLUMES[v]
    m = re.fullmatch(r"([+-]?)" + _NUM + "dB", v)
    if m:
        return float(m.group(1) + m.group(2))
    raise _bad(node, "volume", value, "use +-NdB or silent, x-soft .. x-loud")


def language_of(node: _Node, tag: str) -> str:
    primary = tag.strip().split("-")[0].split("_")[0].lower()
    if primary not in LANGUAGES:
        raise _bad(node, "xml:lang", tag, f"the languages are {', '.join(LANGUAGES)}")
    return LANGUAGES[primary]


def parse(ssml: str, voices: Mapping[str, dict], voice: Optional[str] = None, language: str = "Auto",
          max_segment_chars: int = 400) -> Document:
    """the segments and break plan of an SSML document (module docstring); ValueError names what is refused"""
    from .join import BREAK_MAX_MS
    from .resample import check_prosody
    from .segment import check_max_chars, split_text
    check_max_chars(max_segment_chars)
    if voice is not None and voice not in voices:
        raise ValueError(f"SSML: the default voice {voice!r} is not configured; the voices are {sorted(voices)}")
    root = _parse_xml(ssml)
    spans: List[Span] = []
    breaks: List[Optional[int]] = []
    pending: List[Optional[int]] = [None]            # the breaks at the boundary after the last segment so far
    run: List = [None, []]                           # (context, text pieces) of the current run

    def flush():
        ctx, pieces = run
        run[0], run[1] = None, []
        if ctx is None:
            return
        (voice_name, lang_tag, speed, pitch, gain, lang_node, span_node) = ctx
        texts = split_text(re.sub(r"\s+", " ", "".join(pieces)), max_segment_chars)
        if not texts:
            return
        try:
            check_prosody(speed, pitch, gain)
        except ValueError as ex:
            raise ValueError(f"SSML: the span of <{span_node.tag}> at {span_node.where} composes to rate {speed:g}, "
                             f"pitch {pitch:g} st, volume {gain:g} dB: {ex}") from None
        lang = language_of(lang_node, lang_tag) if lang_tag is not None else voices[voice_name].get("language", language)
        for t in texts:
            breaks.append(pending[0])
            pending[0] = None
            spans.append(Span(t, voice_name, lang, speed, pitch, gain))

    def walk(node: _Node, ctx):
        allowed = ATTRIBUTES.get(node.tag)
        if allowed is None:
            raise ValueError(f"SSML: the element <{node.tag}> is not accepted ({node.where})")
        if node is not root and node.tag == "speak":
            raise ValueError(f"SSML: <speak> is only the root element ({node.where})")
        for name, value in node.attrs.items():
            if name not in allowed:
                raise ValueError(f"SSML: <{node.tag}> attribute {name!r} is not accepted ({node.where})")
        voice_name, lang_tag, speed, pitch, gain, lang_node, span_node = ctx
        if "xml:lang" in node.attrs:
            lang_tag, lang_node = node.attrs["xml:lang"], node
            language_of(node, lang_tag)
        if node.tag == "break":
            if node.children:
                raise ValueError(f"SSML: <break> must be empty ({node.where})")
            flush()
            total = (pending[0] or 0) + break_ms(node)
            if total > BREAK_MAX_MS:
                raise ValueError(f"SSML: the breaks at the boundary of <break> at {node.where} add up to {total} ms, "
                                 f"more than {BREAK_MAX_MS} ms")
            pending[0] = total
            return
        if node.tag == "prosody":
            a = node.attrs
            speed *= rate_factor(node, a["rate"]) if "rate" in a else 1.0
            pitch += pitch_semitones(node, a["pitch"]) if "pitch" in a else 0.0
            gain += volume_db(node, a["volume"]) if "volume" in a else 0.0
            span_node = node
        if node.tag == "voice":
            if "name" not in node.attrs:
                raise ValueError(f"SSML: <voice> needs a name ({node.where})")
            voice_name = node.attrs["name"]
            if voice_name not in voices:
                raise ValueError(f"SSML: <voice> name {voice_name!r} is not configured; the voices are "
                                 f"{sorted(voices)} ({node.where})")
            span_node = node
        if node.tag == "sub":
            if "alias" not in node.attrs:
                raise ValueError(f"SSML: <sub> needs an alias ({node.where})")
            if any(isinstance(c, _Node) for c in node.children):
                raise ValueError(f"SSML: <sub> must hold text only ({node.where})")
            children = [node.attrs["alias"]]
        else:
            children = node.children
        cut = node.tag in ("p", "s")
        if cut:
            flush()
        inner = (voice_name, lang_tag, speed, pitch, gain, lang_node, span_node)
        for c in children:
            if isinstance(c, _Node):
                walk(c, inner)
            elif not c.strip():   # whitespace does not start a run
                if run[0] is not None:
                    run[1].append(c)
            else:
                if voice_name is None:
                    raise ValueError(f"SSML: text outside <voice> needs a default voice ({node.where})")
                if run[0] is not None and run[0][:5] != inner[:5]:
                    flush()
                run[0] = run[0] or inner
                run[1].append(c)
        if cut:
            flush()

    walk(root, (voice, None, 1.0, 0.0, 0.0, None, root))
    flush()
    if not spans:
        raise ValueError("SSML: the document has no text to speak")
    breaks.append(pending[0])
    return Document(spans, breaks)


def voice_request(model, spec: Mapping, text: str, language: Optional[str] = None, split: bool = False,
                  max_segment_chars: int = 400):
    """The ``prepare`` callable (``Segments`` with ``split=True``) of ``text`` spoken by one voice spec -- the dict
    format of the example server's ``--voices`` file: exactly one of ``ref_audio`` (a clone, with optional ``ref_text``
    and ``xvec_only``), ``speaker`` (a custom voice, with optional ``instruct``) or ``design`` (a voice design), and
    optional ``language`` (``language`` overrides it; default ``"Auto"``) and ``max_new_tokens`` (read by the caller).
    The checkpoint's own rules refuse a kind it cannot speak."""
    from . import serving
    kinds = [k for k in ("ref_audio", "speaker", "design") if k in spec]
    if len(kinds) != 1:
        raise ValueError(f"a voice spec holds exactly one of ref_audio, speaker or design, got {sorted(spec)}")
    lang = language if language is not None else spec.get("language", "Auto")
    kw = dict(split=True, max_segment_chars=max_segment_chars) if split else {}
    if kinds[0] == "ref_audio":
        if spec.get("xvec_only"):
            kw["xvec_only"] = True
        return serving.voice_clone_request(model, text, lang, spec["ref_audio"], spec.get("ref_text", ""), **kw)
    if kinds[0] == "speaker":
        return serving.custom_voice_request(model, text, spec["speaker"], lang, instruct=spec.get("instruct"), **kw)
    return serving.custom_voice_request(model, text, None, lang, instruct=spec["design"], **kw)

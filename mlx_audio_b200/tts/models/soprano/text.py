"""Soprano's text normalisation (reference: tts/models/soprano/text.py), restated stdlib-only.

``clean_text`` runs, in order: NFKD to ASCII, numbers, abbreviations, special characters, lower case, removal of characters outside
the model's alphabet, whitespace collapsing, punctuation de-duplication.  Every rule reproduces the reference string for string
(tests/golden/soprano_golden.npz), including its oddities: ``101st`` reads "one hundred oneth", a run of dots becomes a single ".",
and ``#`` is dropped unless a digit follows it.
"""
from __future__ import annotations

import re
import unicodedata

_SMALL = ("zero one two three four five six seven eight nine ten eleven twelve thirteen fourteen fifteen sixteen seventeen "
          "eighteen nineteen").split()
_DECADES = {2: "twenty", 3: "thirty", 4: "forty", 5: "fifty", 6: "sixty", 7: "seventy", 8: "eighty", 9: "ninety"}
_NTH = dict(enumerate(("first second third fourth fifth sixth seventh eighth ninth tenth eleventh twelfth thirteenth fourteenth "
                       "fifteenth sixteenth seventeenth eighteenth nineteenth").split(), start=1))
_NTH.update({10 * k: w[:-1] + "ieth" for k, w in _DECADES.items()})
_SCALES = ((10 ** 9, "billion"), (10 ** 6, "million"), (1000, "thousand"), (100, "hundred"))


def _num_to_words(n: int) -> str:
    """Cardinal words; negatives read "minus ...", numbers past a billion nest ("one thousand billion")."""
    if n < 0:
        return "minus " + _num_to_words(-n)
    if n < 20:
        return _SMALL[n]
    if n < 100:
        tens, ones = divmod(n, 10)
        return _DECADES[tens] + (" " + _SMALL[ones] if ones else "")
    for size, name in _SCALES:
        if n >= size:
            head, rest = divmod(n, size)
            return f"{_num_to_words(head)} {name}" + (" " + _num_to_words(rest) if rest else "")
    raise AssertionError(n)


def _ordinal_to_words(n: int) -> str:
    """Ordinal words: exact below 100; from 100 on the cardinal with "th" appended ("y" -> "ieth")."""
    if n in _NTH:
        return _NTH[n]
    if n < 100:
        tens, ones = divmod(n, 10)
        decade = _DECADES.get(tens, "")
        if not ones:
            return decade + "th"
        return decade + " " + _NTH[ones]
    words = _num_to_words(n)
    return words[:-1] + "ieth" if words.endswith("y") else words + "th"


# ---- abbreviations: dotted ones case-insensitively at a word start, the cased ones as whole words; applied in this order
_DOTTED = (("mrs", "misuss"), ("ms", "miss"), ("mr", "mister"), ("dr", "doctor"), ("st", "saint"), ("co", "company"), ("jr", "junior"),
           ("maj", "major"), ("gen", "general"), ("drs", "doctors"), ("rev", "reverend"), ("lt", "lieutenant"), ("hon", "honorable"),
           ("sgt", "sergeant"), ("capt", "captain"), ("esq", "esquire"), ("ltd", "limited"), ("col", "colonel"), ("ft", "fort"))
_CASED = (("TTS", "text to speech"), ("Hz", "hertz"), ("kHz", "kilohertz"), ("KBs", "kilobytes"), ("KB", "kilobyte"),
          ("MBs", "megabytes"), ("MB", "megabyte"), ("GBs", "gigabytes"), ("GB", "gigabyte"), ("TBs", "terabytes"), ("TB", "terabyte"),
          ("APIs", "a p i's"), ("API", "a p i"), ("CLIs", "c l i's"), ("CLI", "c l i"), ("CPUs", "c p u's"), ("CPU", "c p u"),
          ("GPUs", "g p u's"), ("GPU", "g p u"), ("Ave", "avenue"), ("etc", "etcetera"))
_ABBREVIATIONS = ([(re.compile(rf"\b{a}\.", re.IGNORECASE), w) for a, w in _DOTTED]
                  + [(re.compile(rf"\b{a}\b"), w) for a, w in _CASED])


def expand_abbreviations(text: str) -> str:
    for pattern, words in _ABBREVIATIONS:
        text = pattern.sub(words, text)
    return text


# ---- numbers
_MULTIPLIERS = {"K": "thousand", "M": "million", "B": "billion", "T": "trillion"}


def _plural(n: int, unit: str) -> str:
    return f"{_num_to_words(n)} {unit}" + ("" if n == 1 else "s")


def _money(m) -> str:
    amount = m.group(1).replace(",", "")
    parts = amount.split(".")
    if len(parts) > 2:
        return amount + " dollars"
    dollars = int(parts[0] or 0)
    cents = int(parts[1]) if len(parts) == 2 and parts[1] else 0
    said = [_plural(v, unit) for v, unit in ((dollars, "dollar"), (cents, "cent")) if v]
    return ", ".join(said) if said else "zero dollars"


def _cardinal(m) -> str:
    n = int(m.group(0))
    if not 1000 < n < 3000:
        return _num_to_words(n)
    century, rest = divmod(n, 100)
    if n == 2000:
        return "two thousand"
    if 2000 < n < 2010:
        return "two thousand " + _num_to_words(rest)
    if rest == 0:
        return _num_to_words(century) + " hundred"
    return _num_to_words(century) + (" oh " if rest < 10 else " ") + _num_to_words(rest)


_NUMBER_RULES = (
    (re.compile(r"#\d"), lambda m: "number " + m.group(0)[1]),
    (re.compile(r"\d(K|M|B|T)", re.IGNORECASE), lambda m: f"{m.group(0)[0]} {_MULTIPLIERS[m.group(1).upper()]}"),
    (re.compile(r"(\d[\d,]+\d)"), lambda m: m.group(1).replace(",", "")),
    (re.compile(r"\$([\d.,]*\d+)"), _money),
    (re.compile(r"\d+(st|nd|rd|th)"), lambda m: _ordinal_to_words(int(m.group(0)[:-2]))),
    (re.compile(r"\d+"), _cardinal),
)


def normalize_numbers(text: str) -> str:
    for pattern, fn in _NUMBER_RULES:
        text = pattern.sub(fn, text)
    return text


# ---- characters
_SPECIAL = (("@", " at "), ("&", " and "), ("%", " percent "), (":", "."), (";", ","), ("+", " plus "), ("\\", " backslash "),
            ("~", " about "), ("<", " less than "), (">", " greater than "), ("=", " equals "), ("/", " slash "), ("_", " "))


def expand_special_characters(text: str) -> str:
    for ch, words in _SPECIAL:
        text = text.replace(ch, words)
    return text


def lowercase(text: str) -> str:
    return text.lower()


def convert_to_ascii(text: str) -> str:
    return unicodedata.normalize("NFKD", text).encode("ascii", "ignore").decode("ascii")


_UNKNOWN = re.compile(r"[^A-Za-z !$%&'*+,\-./0-9<>?_]")
_DROPPED = re.compile(r"[<>/_+]")


def remove_unknown_characters(text: str) -> str:
    return _DROPPED.sub("", _UNKNOWN.sub("", text))


def collapse_whitespace(text: str) -> str:
    text = re.sub(r"\s+", " ", text)
    return re.sub(r" ([.?!,])", r"\1", text).strip()


_PUNCT_RULES = ((re.compile(r"\.{3,}"), "..."), (re.compile(r",+"), ","), (re.compile(r"[.,]*\.[.,]*"), "."),
                (re.compile(r"[.,!]*![.,!]*"), "!"), (re.compile(r"[.,!?]*\?[.,!?]*"), "?"))


def dedup_punctuation(text: str) -> str:
    for pattern, repl in _PUNCT_RULES:
        text = pattern.sub(repl, text)
    return text


_PIPELINE = (convert_to_ascii, normalize_numbers, expand_abbreviations, expand_special_characters, lowercase, remove_unknown_characters,
             collapse_whitespace, dedup_punctuation)


def clean_text(text: str) -> str:
    """Normalise ``text`` for Soprano's tokenizer (the reference's clean_text)."""
    for step in _PIPELINE:
        text = step(text)
    return text

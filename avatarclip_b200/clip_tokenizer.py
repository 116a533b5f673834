"""openai/CLIP's byte-level BPE tokenizer (``clip.tokenize``, AvatarGen/AppearanceGen/main.py:274,280,286), restated
from its published description so that the prompts can be encoded without the ``clip`` package.

The merges come from openai's ``bpe_simple_vocab_16e6.txt.gz`` (shipped inside the ``clip`` package, not inside
``ViT-B-32.pt``).  With that file, ``ClipTokenizer(path).tokenize("a photo of a cat")`` gives
``[49406, 320, 1125, 539, 320, 2368, 49407, 0, ...]``.

* Vocabulary order: the 256 byte symbols, the same with ``</w>`` appended, one symbol per merge (lines
  ``[1 : 49152-256-2+1]`` of the file: the first line is a version header), ``<|startoftext|>``, ``<|endoftext|>``.
* Cleaning: ``html.unescape`` twice, whitespace runs collapsed to one space, stripped, lowercased.  openai also runs
  ``ftfy.fix_text`` first.  ftfy is not a dependency here and it leaves ASCII text unchanged; every prompt of the
  shipped confs is ASCII.  Non-ASCII text that ftfy would repair may therefore tokenize differently.
* Pre-tokenizer: openai's regular expression (the ``regex`` package, for ``\\p{L}`` / ``\\p{N}``); each piece is
  UTF-8 encoded, mapped through the byte-to-unicode table and merged lowest rank first.
"""
from __future__ import annotations

import functools
import gzip
import html
from typing import Dict, List, Sequence, Tuple, Union

import regex
import torch

SOT, EOT = "<|startoftext|>", "<|endoftext|>"
N_MERGES = 49152 - 256 - 2          # merges lines [1 : N_MERGES + 1]: the vocabulary is 512 + 48894 + 2 = 49408
_PATTERN = regex.compile(r"<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+",
                         regex.IGNORECASE)


@functools.lru_cache(maxsize=None)
def bytes_to_unicode() -> Dict[int, str]:
    """Byte -> printable unicode character: the 188 printable Latin-1 bytes map to themselves, the other 68 bytes to
    U+0100 onwards in byte order (so no symbol is whitespace or a control character).  The dict lists the printable
    bytes first: that is the order of the first 256 vocabulary entries ("!" = 0, "a" = 64)."""
    keep = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    table = {b: chr(b) for b in keep}
    for b in range(256):
        if b not in table:
            table[b] = chr(256 + len(table) - len(keep))
    return table


def clean(text: str) -> str:
    """HTML entities unescaped twice ("&amp;amp;" -> "&"), whitespace collapsed and stripped, lowercased."""
    text = html.unescape(html.unescape(text)).strip()
    return regex.sub(r"\s+", " ", text).strip().lower()


def read_merges(bpe_path: str) -> List[Tuple[str, str]]:
    with gzip.open(bpe_path, "rt", encoding="utf-8") as f:
        lines = f.read().split("\n")[1:N_MERGES + 1]
    return [tuple(line.split()) for line in lines if line.strip()]


class ClipTokenizer:
    def __init__(self, bpe_path: str):
        self.merges = read_merges(bpe_path)
        self.ranks = {m: i for i, m in enumerate(self.merges)}
        byte_syms = list(bytes_to_unicode().values())
        vocab = byte_syms + [s + "</w>" for s in byte_syms] + ["".join(m) for m in self.merges] + [SOT, EOT]
        self.encoder = {s: i for i, s in enumerate(vocab)}
        self.sot, self.eot = self.encoder[SOT], self.encoder[EOT]
        self._cache = {}

    def _bpe(self, piece: str) -> List[str]:
        """Merge the symbols of one pre-tokenized piece (the last symbol carries ``</w>``), lowest merge rank first."""
        if piece in self._cache:
            return self._cache[piece]
        word = list(piece[:-1]) + [piece[-1] + "</w>"]
        while len(word) > 1:
            pairs = {(word[i], word[i + 1]) for i in range(len(word) - 1)}
            best = min(pairs, key=lambda p: self.ranks.get(p, float("inf")))
            if best not in self.ranks:
                break
            merged, i = [], 0
            while i < len(word):
                if i + 1 < len(word) and (word[i], word[i + 1]) == best:
                    merged.append(word[i] + word[i + 1])
                    i += 2
                else:
                    merged.append(word[i])
                    i += 1
            word = merged
        self._cache[piece] = word
        return word

    def encode(self, text: str) -> List[int]:
        """Token ids of ``text`` without the start / end tokens."""
        table = bytes_to_unicode()
        ids = []
        for piece in _PATTERN.findall(clean(text)):
            piece = "".join(table[b] for b in piece.encode("utf-8"))
            ids.extend(self.encoder[s] for s in self._bpe(piece))
        return ids

    def tokenize(self, texts: Union[str, Sequence[str]], context_length: int = 77, truncate: bool = False) -> torch.Tensor:
        """``clip.tokenize``: int32 [N, context_length], each row <|startoftext|> ids <|endoftext|> then zeros.  A text
        that does not fit raises RuntimeError; with ``truncate`` it is cut and its last position set to <|endoftext|>."""
        if isinstance(texts, str):
            texts = [texts]
        out = torch.zeros(len(texts), context_length, dtype=torch.int32)
        for i, text in enumerate(texts):
            ids = [self.sot] + self.encode(text) + [self.eot]
            if len(ids) > context_length:
                if not truncate:
                    raise RuntimeError(f"Input {text} is too long for context length {context_length}")
                ids = ids[:context_length]
                ids[-1] = self.eot
            out[i, :len(ids)] = torch.tensor(ids, dtype=torch.int32)
        return out

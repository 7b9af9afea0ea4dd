"""Text tokenizer wrapper (reference tokenizer.py:12-38): a HF tokenizer shipped in the model snapshot, ids
wrapped in BOS/EOS.  ``IdsTokenizer`` is the offline stand-in for synthetic checkpoints: whitespace-separated
integer ids, or a deterministic hash of each word into the vocabulary."""
from __future__ import annotations

import re
import zlib
from typing import List, Optional, Tuple

Span = Optional[Tuple[int, int]]


class TextTokenizer:
    def __init__(self, model_name: str, add_bos_eos: bool = True):
        from transformers import AutoTokenizer

        self.tok = AutoTokenizer.from_pretrained(model_name, use_fast=True)
        self.add_bos_eos = add_bos_eos
        if self.tok.pad_token_id is None:
            self.tok.add_special_tokens({"pad_token": "<|pad|>"})
        self.pad_id = int(self.tok.pad_token_id)
        self.bos_id = None if self.tok.bos_token_id is None else int(self.tok.bos_token_id)
        self.eos_id = None if self.tok.eos_token_id is None else int(self.tok.eos_token_id)
        self.vocab_size = int(self.tok.vocab_size + len(self.tok.get_added_vocab()))

    def encode(self, text: str) -> List[int]:
        ids = self.tok.encode(text, add_special_tokens=False)
        if self.add_bos_eos and self.bos_id is not None and self.eos_id is not None:
            ids = [self.bos_id] + ids + [self.eos_id]
        return ids

    def encode_with_offsets(self, text: str) -> Tuple[List[int], List[Span]]:
        """(encode(text), the (start, end) character span of each id in `text`; BOS and EOS have none).  Raises when
        the offsets pass of the fast tokenizer gives other ids than encode, rather than guessing."""
        enc = self.tok(text, add_special_tokens=False, return_offsets_mapping=True)
        ids = [int(i) for i in enc["input_ids"]]
        spans: List[Span] = [(int(a), int(b)) for a, b in enc["offset_mapping"]]
        if self.add_bos_eos and self.bos_id is not None and self.eos_id is not None:
            ids = [self.bos_id] + ids + [self.eos_id]
            spans = [None] + spans + [None]
        if ids != self.encode(text):
            raise ValueError("the tokenizer's offsets pass gives other ids than encode(); cannot map tokens to characters")
        return ids, spans


class IdsTokenizer:
    def __init__(self, vocab_size: int, add_bos_eos: bool = True):
        self.vocab_size = int(vocab_size)
        self.add_bos_eos = add_bos_eos
        self.bos_id, self.eos_id, self.pad_id = self.vocab_size - 2, self.vocab_size - 1, 0

    def encode(self, text: str) -> List[int]:
        ids = []
        for w in text.split():
            ids.append(int(w) % (self.vocab_size - 2) if w.lstrip("-").isdigit() else zlib.crc32(w.encode()) % (self.vocab_size - 2))
        return [self.bos_id] + ids + [self.eos_id] if self.add_bos_eos else ids

    def encode_with_offsets(self, text: str) -> Tuple[List[int], List[Span]]:
        """(encode(text), the (start, end) character span of each id in `text`; BOS and EOS have none)."""
        spans: List[Span] = [(m.start(), m.end()) for m in re.finditer(r"\S+", text)]
        if self.add_bos_eos:
            spans = [None] + spans + [None]
        return self.encode(text), spans

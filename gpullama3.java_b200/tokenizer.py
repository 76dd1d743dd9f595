"""Host mirror of the reference's tokenizers over the native byte-level BPE (csrc/tokenizer.cpp, include/b200tok.h).

``Tokenizer`` <- tokenizer/Tokenizer.java (interface), ``LlamaTokenizer`` <- tokenizer/LlamaTokenizer.java:30-269,
``Qwen3Tokenizer`` <- tokenizer/Qwen3Tokenizer.java:20-352; ``Vocabulary.loadLlamaVocabulary`` reads
``tokenizer.ggml.tokens`` / ``tokenizer.ggml.merges`` (/ ``token_type``) from the GGUF metadata.  The hot part
(byte mapping, pre-tokenisation, merge loop, byte decoding) is native; special-token bookkeeping stays here.
There is no Python fallback: a missing libb200tok.so raises."""
from __future__ import annotations

import ctypes as C
import os
import re

from . import build as _build

KIND_LLAMA3, KIND_QWEN3 = 0, 1
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    path = _build.build_tokenizer()
    L = C.CDLL(path)
    vp, i32, sz = C.c_void_p, C.c_int32, C.c_size_t
    L.b200_tok_create.argtypes = [C.POINTER(C.c_char_p), i32, C.POINTER(C.c_char_p), i32, i32, C.POINTER(vp), C.c_char_p, sz]
    L.b200_tok_encode.argtypes = [vp, C.c_char_p, sz, C.POINTER(i32), sz, C.POINTER(sz)]
    L.b200_tok_encode_mapped.argtypes = [vp, C.c_char_p, sz, C.POINTER(i32), sz, C.POINTER(sz)]
    L.b200_tok_decode.argtypes = [vp, C.POINTER(i32), sz, C.c_char_p, sz, C.POINTER(sz)]
    L.b200_tok_split.argtypes = [i32, C.c_char_p, sz, C.POINTER(i32), sz, C.POINTER(sz)]
    L.b200_tok_index.argtypes = [vp, C.c_char_p]
    L.b200_tok_index.restype = i32
    L.b200_tok_vocab_size.argtypes = [vp]
    L.b200_tok_vocab_size.restype = i32
    L.b200_tok_free.argtypes = [vp]
    L.b200_tok_free.restype = None
    _lib = L
    return L


EXPORTS = ["b200_tok_create", "b200_tok_encode", "b200_tok_encode_mapped", "b200_tok_decode", "b200_tok_split", "b200_tok_index", "b200_tok_vocab_size", "b200_tok_free"]


def split_lengths(data: bytes, kind: int = KIND_LLAMA3) -> list[int]:
    """Byte lengths of the pre-tokenisation chunks (test hook)."""
    cap = len(data) + 1
    buf = (C.c_int32 * cap)()
    n = C.c_size_t(0)
    rc = lib().b200_tok_split(kind, data, len(data), buf, cap, C.byref(n))
    if rc != 0:
        raise TokenizerError(f"b200_tok_split failed ({rc})")
    return list(buf[: n.value])


class TokenizerError(RuntimeError):
    pass


class Tokenizer:
    """Common part of LlamaTokenizer / Qwen3Tokenizer."""

    kind = KIND_LLAMA3

    def __init__(self, tokens: list[str], merge_lines: list[str], base_tokens: int, token_types: list[int] | None = None):
        self.tokens = list(tokens)
        self.token_types = token_types
        L = lib()
        tarr = (C.c_char_p * len(tokens))(*[t.encode("utf-8") for t in tokens])
        marr = (C.c_char_p * max(1, len(merge_lines)))(*[m.encode("utf-8") for m in merge_lines])
        h = C.c_void_p()
        err = C.create_string_buffer(512)
        rc = L.b200_tok_create(tarr, len(tokens), marr, len(merge_lines), self.kind, C.byref(h), err, 512)
        if rc != 0:
            raise TokenizerError(f"b200_tok_create failed ({rc}): {err.value.decode()}")
        self._h = h
        # "assume all tokens after the base ones are special" (LlamaTokenizer.java:45-52)
        self.special_tokens = {tokens[i]: i for i in range(base_tokens, len(tokens))}
        self._special_ids = set(self.special_tokens.values())

    def close(self):
        if getattr(self, "_h", None):
            lib().b200_tok_free(self._h)
            self._h = None

    __del__ = close

    # List<Integer> encodeAsList(String text)
    def encode_as_list(self, text: str) -> list[int]:
        return self._call(lib().b200_tok_encode, text.encode("utf-8"))

    encode = encode_as_list

    # List<Integer> encode(String text, Set<String> allowedSpecial) -- text is byte-mapped, as in the reference
    def encode_with_special(self, mapped_text: str, allowed_special: set[str]) -> list[int]:
        if not allowed_special:
            return self._call(lib().b200_tok_encode_mapped, mapped_text.encode("utf-8"))
        missing = [s for s in allowed_special if s not in self.special_tokens]
        if missing:
            raise TokenizerError(f"not special tokens: {missing}")
        # Java's String.split never returns the delimiters, capturing group or not (unlike Python's re.split), and drops
        # trailing empty strings: the reference's encode(text, allowedSpecial) therefore DROPS the special tokens it splits at
        # (its `special.contains(part)` branch is dead code, LlamaTokenizer.java:164-176).  Mirrored as is: chat formats add
        # special tokens by id (LlamaChatFormat.java), never through this path.
        parts = re.split("(?:" + "|".join(re.escape(s) for s in allowed_special) + ")", mapped_text)
        while parts and parts[-1] == "":
            parts.pop()
        ids = []
        for part in parts:
            if part in allowed_special:
                ids.append(self.special_tokens[part])
            else:
                ids.extend(self._call(lib().b200_tok_encode_mapped, part.encode("utf-8")))
        return ids

    def _call(self, fn, data: bytes) -> list[int]:
        cap = len(data) + 8
        buf = (C.c_int32 * cap)()
        n = C.c_size_t(0)
        rc = fn(self._h, data, len(data), buf, cap, C.byref(n))
        if rc == -3:  # cannot happen: a token covers at least one byte
            buf = (C.c_int32 * n.value)()
            rc = fn(self._h, data, len(data), buf, n.value, C.byref(n))
        if rc != 0:
            raise TokenizerError(f"encode failed ({rc}): a symbol of the text has no token in the vocabulary")
        return list(buf[: n.value])

    # String decode(List<Integer> tokens)
    def decode_bytes(self, ids) -> bytes:
        arr = (C.c_int32 * len(ids))(*ids)
        n = C.c_size_t(0)
        rc = lib().b200_tok_decode(self._h, arr, len(ids), None, 0, C.byref(n))
        if rc not in (0, -3):
            raise TokenizerError(f"decode failed ({rc})")
        out = C.create_string_buffer(max(1, n.value))
        rc = lib().b200_tok_decode(self._h, arr, len(ids), out, n.value, C.byref(n))
        if rc != 0:
            raise TokenizerError(f"decode failed ({rc})")
        return out.raw[: n.value]

    def decode(self, ids) -> str:
        return self.decode_bytes(ids).decode("utf-8", errors="replace")  # new String(bytes, UTF_8) replaces malformed input

    def get_special_tokens(self) -> dict[str, int]:
        return self.special_tokens

    def is_special_token(self, token: int) -> bool:
        return token in self._special_ids

    def should_display_token(self, token: int) -> bool:
        return not self.is_special_token(token)

    def index(self, token: str) -> int:
        return lib().b200_tok_index(self._h, token.encode("utf-8"))


class LlamaTokenizer(Tokenizer):
    kind = KIND_LLAMA3
    BASE_TOKENS = 128000  # LlamaTokenizer.java:45

    def __init__(self, tokens, merge_lines, base_tokens: int | None = None):
        super().__init__(tokens, merge_lines, self.BASE_TOKENS if base_tokens is None else base_tokens)


class Qwen3Tokenizer(Tokenizer):
    kind = KIND_QWEN3

    def __init__(self, tokens, merge_lines, token_types, deepseek_r1_distill: bool = False):
        first = "<｜end▁of▁sentence｜>" if deepseek_r1_distill else "<|endoftext|>"  # Qwen3Tokenizer.java:58-60
        super().__init__(tokens, merge_lines, list(tokens).index(first), token_types)
        self.think_start_token = self.special_tokens.pop("<think>", -1)   # :74-79
        self.think_end_token = self.special_tokens.pop("</think>", -1)
        self._special_ids = set(self.special_tokens.values())

    def should_display_token(self, token: int) -> bool:  # :174-178
        return self.token_types[token] in (1, 4, 6)


class UnsupportedTokenizer(Exception):
    """The model's tokenizer family is outside this package's scope (maps to UnsupportedOperationException)."""


def from_metadata(metadata: dict, model_type: str) -> Tokenizer:
    """ModelLoader: Vocabulary.loadLlamaVocabulary / loadQwen3Vocabulary + the tokenizer constructors."""
    if model_type.upper() in ("MISTRAL", "DEVSTRAL_2", "PHI_3", "GRANITE") or "tokenizer.ggml.merges" not in metadata:
        # MistralTokenizer / Phi3Tokenizer (tokenizer/MistralTokenizer.java, Phi3Tokenizer.java) are SentencePiece-style scorers, not the
        # byte-level BPE implemented here; GraniteTokenizer is byte-level BPE with its own pre-tokenisation patterns (REFACT / DBRX, by
        # tokenizer.ggml.pre), which the Llama-3 tokenizer would get wrong.  Reject up front instead of mis-tokenising (the forward
        # pass itself is supported).
        raise UnsupportedTokenizer(f"no tokenizer for model type {model_type}: only the byte-level BPE vocabularies of Llama-3 and Qwen3 are "
                                   "implemented; drive the plan with token ids")
    tokens = list(metadata["tokenizer.ggml.tokens"])
    merges = list(metadata["tokenizer.ggml.merges"])
    typ = model_type.upper()
    if typ.startswith("QWEN") or typ == "DEEPSEEK_R1_DISTILL_QWEN":
        # Qwen2ModelLoader.java:35-43: the Qwen3 vocabulary and tokenizer; DeepSeek-R1-Distill-Qwen moves the first special token
        deepseek = typ != "QWEN_3" and metadata.get("general.basename") == "DeepSeek-R1-Distill-Qwen"
        return Qwen3Tokenizer(tokens, merges, list(metadata["tokenizer.ggml.token_type"]), deepseek_r1_distill=deepseek)
    return LlamaTokenizer(tokens, merges, base_tokens=metadata.get("b200.synthetic.base_tokens"))

"""ctypes driver of the byte-level BPE tokenizer (b200_tokenizer_*, csrc/tokenizer.cc): a local HF tokenizer.json of the
Llama-3 family, the same ids as HF `tokenizers`, and the Llama-3 instruct chat framing."""
from __future__ import annotations

import ctypes as C

from ._lib import check, lib


class Tokenizer:
    def __init__(self, tokenizer_json: str):
        self._l = lib()
        self._h = C.c_void_p()
        check(self._l.b200_tokenizer_load(str(tokenizer_json).encode(), C.byref(self._h)))

    def close(self):
        if self._h:
            self._l.b200_tokenizer_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    @property
    def vocab_size(self) -> int:
        return self._l.b200_tokenizer_vocab_size(self._h)

    def token_id(self, content: str) -> int:
        return self._l.b200_tokenizer_token_id(self._h, content.encode("utf-8"))

    def encode(self, text: str, allow_special: bool = True) -> list:
        b = text.encode("utf-8")
        n = self._l.b200_tokenizer_encode(self._h, b, len(b), 1 if allow_special else 0, None, 0)
        buf = (C.c_int32 * max(int(n), 1))()
        self._l.b200_tokenizer_encode(self._h, b, len(b), 1 if allow_special else 0, buf, n)
        return list(buf[:n])

    def encode_pair(self, query: str, document: str, join: bool = False, add_special_tokens: bool = True) -> list:
        """A score pair's ids (b200_tokenizer_encode_pair): join False = HF tokenizer(text=query, text_pair=document),
        True = tokenizer(text=query + document)."""
        a, b = query.encode("utf-8"), document.encode("utf-8")
        args = (self._h, a, len(a), b, len(b), 1 if join else 0, 1 if add_special_tokens else 0)
        n = self._l.b200_tokenizer_encode_pair(*args, None, 0)
        buf = (C.c_int32 * max(n, 1))()
        self._l.b200_tokenizer_encode_pair(*args, buf, n)
        return list(buf[:n])

    def decode(self, ids, skip_special: bool = False) -> str:
        arr = (C.c_int32 * max(len(ids), 1))(*ids)
        n = self._l.b200_tokenizer_decode(self._h, arr, len(ids), 1 if skip_special else 0, None, 0)
        out = C.create_string_buffer(int(n) + 1)
        self._l.b200_tokenizer_decode(self._h, arr, len(ids), 1 if skip_special else 0, out, n + 1)
        return out.raw[:n].decode("utf-8", "replace")

    def chat(self, messages, add_generation_prompt: bool = True) -> list:
        n = len(messages)
        roles = (C.c_char_p * max(n, 1))(*[m["role"].encode("utf-8") for m in messages])
        contents = (C.c_char_p * max(n, 1))(*[m["content"].encode("utf-8") for m in messages])
        k = self._l.b200_tokenizer_chat_llama3(self._h, roles, contents, n, 1 if add_generation_prompt else 0, None, 0)
        if k < 0:
            check(-1)
        buf = (C.c_int32 * max(int(k), 1))()
        self._l.b200_tokenizer_chat_llama3(self._h, roles, contents, n, 1 if add_generation_prompt else 0, buf, k)
        return list(buf[:k])


class DetokStream:
    """Incremental detokenisation (b200_tokenizer_stream_*): push(id) returns the text that id completed."""

    def __init__(self, tokenizer: Tokenizer, skip_special: bool = True):
        self._l = lib()
        self._tok = tokenizer
        self._h = self._l.b200_tokenizer_stream_new(tokenizer._h, 1 if skip_special else 0)

    def _call(self, token_id: int) -> str:
        buf = C.create_string_buffer(256)
        n = self._l.b200_tokenizer_stream_push(self._h, token_id, buf, len(buf))
        assert 0 <= n < len(buf)
        return buf.raw[:n].decode("utf-8")        # strict: a push never returns a broken sequence

    def push(self, token_id: int) -> str:
        return self._call(token_id)

    def flush(self) -> str:
        return self._call(-1)

    def close(self):
        if self._h:
            self._l.b200_tokenizer_stream_free(self._h)
            self._h = None

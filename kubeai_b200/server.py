"""ctypes driver of the serving shell and the load generator (b200_server_*, b200_harness_*).
Shaped like the reference: Server.handle() is modelproxy.Handler.ServeHTTP with a ResponseWriter,
Harness mirrors benchmarks/multi-turn-chat-go's Config/Result."""
from __future__ import annotations

import ctypes as C
import json

from ._lib import (BEGIN_FN, WRITE_FN, HarnessConfig, HarnessResult, ResponseWriter, ServerConfig, check, lib)

LEAST_LOAD, PREFIX_HASH = 0, 1


def tokenize(text: str, vocab: int = 128256) -> list:
    b = text.encode("utf-8")
    n = lib().b200_tokenize(vocab, b, len(b), None, 0)
    buf = (C.c_int32 * max(n, 1))()
    lib().b200_tokenize(vocab, b, len(b), buf, n)
    return list(buf[:n])


def detokenize(ids, vocab: int = 128256) -> str:
    arr = (C.c_int32 * max(len(ids), 1))(*ids)
    n = lib().b200_detokenize(vocab, arr, len(ids), None, 0)
    out = C.create_string_buffer(n + 1)
    lib().b200_detokenize(vocab, arr, len(ids), out, n + 1)
    return out.value.decode("utf-8", "replace")


class Response:
    def __init__(self):
        self.status, self.content_type, self.body = 0, "", b""

    def json(self):
        return json.loads(self.body)

    def sse_events(self):
        return [e[6:] for e in self.body.decode().split("\n\n") if e.startswith("data: ")]


class Server:
    """enable_sampling: serve requests with temperature >= 1e-5 (temperature / top_p / top_k / seed); off, they get a 400
    and the server decodes greedily only (the serving shell's behaviour before sampling existed).
    enable_logprobs: serve logprobs / top_logprobs in vLLM's response format; off, they get a 400.
    enable_logits_processors: serve presence / frequency / repetition penalties, min_p, min_tokens and logit_bias; off,
    they get a 400.
    enable_prompt_logprobs: serve prompt_logprobs (both routes) and echo (completions) in vLLM's response format; off,
    they get a 400.
    max_n: k >= 2 serves "n" up to k (parallel sampling, at most the engines' max_num_seqs); 0 or 1, n > 1 gets a 400."""

    def __init__(self, engines, model="llama-3-8b", adapters=None, strategy=LEAST_LOAD, mean_load_pct=125,
                 replication=256, prefix_char_length=100, max_retries=3, default_max_tokens=256, vocab=128256,
                 max_model_len=2048, enable_sampling=False, enable_logprobs=False, enable_logits_processors=False,
                 enable_prompt_logprobs=False, max_n=0):
        self._l = lib()
        self._engines = list(engines)   # keep alive; entries may be None for parse-path-only tests
        n = len(self._engines)
        arr = (C.c_void_p * n)(*[(e._h if e is not None else None) for e in self._engines])
        cfg = ServerConfig(model=model.encode(), adapters=",".join(adapters).encode() if adapters else None,
                           strategy=strategy, mean_load_pct=mean_load_pct, replication=replication,
                           prefix_char_length=prefix_char_length, max_retries=max_retries,
                           default_max_tokens=default_max_tokens, vocab=vocab, max_model_len=max_model_len,
                           enable_sampling=1 if enable_sampling else 0,
                           enable_logprobs=1 if enable_logprobs else 0,
                           enable_logits_processors=1 if enable_logits_processors else 0,
                           enable_prompt_logprobs=1 if enable_prompt_logprobs else 0, max_n=max_n)
        self._h = C.c_void_p()
        check(self._l.b200_server_create(C.byref(cfg), arr, n, C.byref(self._h)))

    def close(self):
        if self._h:
            self._l.b200_server_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def handle(self, method: str, path: str, body: bytes | str = b"", content_type: str = "application/json",
               on_chunk=None) -> Response:
        if isinstance(body, str):
            body = body.encode("utf-8")
        resp = Response()

        def begin(_ud, status, ctype):
            resp.status, resp.content_type = status, (ctype or b"").decode()
            return 0

        def write(_ud, data, n):
            chunk = C.string_at(data, n)
            resp.body += chunk
            return 1 if (on_chunk and on_chunk(chunk)) else 0

        w = ResponseWriter(None, BEGIN_FN(begin), WRITE_FN(write))
        st = self._l.b200_server_handle(self._h, method.encode(), path.encode(), content_type.encode(), body,
                                        len(body), C.byref(w))
        if resp.status == 0:
            resp.status = st
        return resp

    def parse_request(self, path: str, body: bytes | str, content_type: str = "application/json", prefix_chars: int = -1):
        """(status, dict) of apiutils.ParseRequest; status 0 on success."""
        if isinstance(body, str):
            body = body.encode("utf-8")
        out = C.create_string_buffer(1 << 16)
        st = self._l.b200_server_parse_request(self._h, path.encode(), content_type.encode(), body, len(body),
                                               prefix_chars, out, len(out))
        return st, json.loads(out.value)

    def listen(self, host="127.0.0.1", port=0) -> int:
        bound = C.c_int32()
        check(self._l.b200_server_listen(self._h, host.encode(), port, C.byref(bound)))
        return bound.value

    def metrics(self) -> str:
        buf = C.create_string_buffer(1 << 16)
        check(self._l.b200_server_metrics(self._h, buf, len(buf)))
        return buf.value.decode()

    def set_tokenizer(self, tokenizer):
        """Attach a kubeai_b200.tokenizer.Tokenizer (or None): Llama-3 chat framing, eot stop ids, incremental detokenisation."""
        self._tokenizer = tokenizer          # keep alive: the server does not own it
        check(self._l.b200_server_set_tokenizer(self._h, tokenizer._h if tokenizer is not None else None))

    def render_prompt(self, path: str, body: bytes | str, content_type: str = "application/json") -> list:
        """The token ids the server would submit for this request (host-only)."""
        if isinstance(body, str):
            body = body.encode("utf-8")
        n = self._l.b200_server_render_prompt(self._h, path.encode(), content_type.encode(), body, len(body), None, 0)
        if n < 0:
            check(-1)
        buf = (C.c_int32 * max(int(n), 1))()
        self._l.b200_server_render_prompt(self._h, path.encode(), content_type.encode(), body, len(body), buf, n)
        return list(buf[:n])

    def inject_fault(self, replica: int, count: int):
        check(self._l.b200_server_inject_fault(self._h, replica, count))


def harness_config(**kw) -> HarnessConfig:
    cfg = HarnessConfig()
    lib().b200_harness_config_default(C.byref(cfg))
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise AttributeError(k)
        setattr(cfg, k, v.encode() if isinstance(v, str) else v)
    return cfg


def synth_threads(cfg: HarnessConfig) -> list:
    n = lib().b200_harness_synth_threads(C.byref(cfg), None, 0)
    buf = C.create_string_buffer(n + 1)
    lib().b200_harness_synth_threads(C.byref(cfg), buf, n + 1)
    return json.loads(buf.value)


def harness_run(cfg: HarnessConfig, server: Server | None = None, host: str | None = None, port: int = 0,
                threads=None) -> dict:
    res = HarnessResult()
    tj = json.dumps(threads).encode() if threads is not None else None
    check(lib().b200_harness_run(server._h if server else None, host.encode() if host else None, port,
                                 C.byref(cfg), tj, len(tj) if tj else 0, C.byref(res)))
    return res.as_dict()

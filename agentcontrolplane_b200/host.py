"""ctypes binding of include/acp_host.h (libacp_host.so) — the C++ host mirror of the reference's Go code on the
path (llmclient + Task LLM step) and the reconcile-loop simulator.  JSON in, JSON out."""
from __future__ import annotations

import ctypes
import json
from typing import Any

from . import _lib

_bound = None


def lib():
    global _bound
    if _bound is None:
        l = _lib.load_host()
        cp, vp = ctypes.c_char_p, ctypes.c_void_p
        out = ctypes.POINTER(ctypes.c_void_p)
        l.acp_host_render_prompt.argtypes = [cp, ctypes.c_size_t, out]
        l.acp_host_parse_completion.argtypes = [cp, ctypes.c_size_t, cp, cp, out]
        l.acp_host_decode_tokens.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.c_int, out,
                                             ctypes.POINTER(ctypes.c_size_t)]
        l.acp_host_build_chat_request.argtypes = [cp, cp, cp, out]
        l.acp_host_convert_response.argtypes = [cp, out]
        l.acp_host_task_step.argtypes = [vp, cp, out]
        l.acp_host_stub_server_start.argtypes = [cp, ctypes.POINTER(ctypes.c_int)]
        l.acp_host_stub_server_stop.argtypes = [ctypes.c_int]
        l.acp_host_stub_server_stop.restype = None
        l.acp_hostsim_run.argtypes = [vp, cp, out]
        l.acp_host_checkpoint_index.argtypes = [cp, out]
        l.acp_host_model_preset.argtypes = [cp, out]
        l.acp_host_free.argtypes = [vp]
        l.acp_host_free.restype = None
        _bound = l
    return _bound


def _take(buf, length=None) -> bytes:
    try:
        return ctypes.string_at(buf) if length is None else ctypes.string_at(buf, length)
    finally:
        lib().acp_host_free(buf)


def _check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed with ACP error {rc}")


def render_prompt(request: dict) -> dict:
    body = json.dumps(request).encode()
    buf = ctypes.c_void_p()
    _check(lib().acp_host_render_prompt(body, len(body), ctypes.byref(buf)), "acp_host_render_prompt")
    return json.loads(_take(buf))


def parse_completion(text: str | bytes, tools: list | None, prefix: str = "call_") -> dict:
    raw = text if isinstance(text, bytes) else text.encode()
    buf = ctypes.c_void_p()
    _check(lib().acp_host_parse_completion(raw, len(raw), json.dumps(tools or []).encode(),
                                           prefix.encode(), ctypes.byref(buf)), "acp_host_parse_completion")
    return json.loads(_take(buf))


def decode_tokens(ids: list[int]) -> bytes:
    arr = (ctypes.c_int * len(ids))(*ids)
    buf, ln = ctypes.c_void_p(), ctypes.c_size_t(0)
    _check(lib().acp_host_decode_tokens(arr, len(ids), ctypes.byref(buf), ctypes.byref(ln)),
           "acp_host_decode_tokens")
    return _take(buf, ln.value)


def build_chat_request(model: str, messages: list, tools: list) -> dict:
    buf = ctypes.c_void_p()
    _check(lib().acp_host_build_chat_request(model.encode(), json.dumps(messages).encode(),
                                             json.dumps(tools).encode(), ctypes.byref(buf)),
           "acp_host_build_chat_request")
    return json.loads(_take(buf))


def convert_response(response: dict | str) -> dict:
    body = response if isinstance(response, str) else json.dumps(response)
    buf = ctypes.c_void_p()
    _check(lib().acp_host_convert_response(body.encode(), ctypes.byref(buf)), "acp_host_convert_response")
    return json.loads(_take(buf))


def task_step(inp: dict, engine=None) -> dict:
    buf = ctypes.c_void_p()
    h = engine._h if engine is not None else None
    _check(lib().acp_host_task_step(h, json.dumps(inp).encode(), ctypes.byref(buf)), "acp_host_task_step")
    return json.loads(_take(buf))


class StubServer:
    """Loopback stub completion server (the reference tests' httptest.NewServer)."""

    def __init__(self, body: str | None = None):
        port = ctypes.c_int(0)
        self.handle = lib().acp_host_stub_server_start(body.encode() if body else None, ctypes.byref(port))
        if self.handle < 0:
            raise RuntimeError("stub server failed to start")
        self.port = port.value
        self.base_url = f"http://127.0.0.1:{self.port}/v1"

    def close(self):
        if self.handle >= 0:
            lib().acp_host_stub_server_stop(self.handle)
            self.handle = -1

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def hostsim_run(config: dict[str, Any], engine=None) -> dict:
    buf = ctypes.c_void_p()
    h = engine._h if engine is not None else None
    _check(lib().acp_hostsim_run(h, json.dumps(config).encode(), ctypes.byref(buf)), "acp_hostsim_run")
    return json.loads(_take(buf))


def hostsim_window_tokens(prompt_tokens: int, tools: int) -> int:
    """Length of the context window hostsim builds for this target (a dry run with zero Tasks)."""
    r = hostsim_run({"tasks": 0, "provider": "openai", "prompt_tokens": prompt_tokens, "tools": tools})
    return int(r["prompt_tokens"])


def checkpoint_index(path: str) -> dict:
    """What acp_infer_init {"weights": path} would see: tensor table, config.json, derived model
    config (raises ValueError with the loader's message when the checkpoint is not usable)."""
    buf = ctypes.c_void_p()
    rc = lib().acp_host_checkpoint_index(path.encode(), ctypes.byref(buf))
    out = json.loads(_take(buf)) if buf.value else {}
    if rc != 0:
        raise ValueError(out.get("error", f"acp_host_checkpoint_index failed with {rc}"))
    return out


def model_preset(name: str) -> dict:
    """The architecture of the engine's synthetic preset `name` (the "model" object of checkpoint_index);
    raises KeyError for a name the engine does not know."""
    buf = ctypes.c_void_p()
    rc = lib().acp_host_model_preset(name.encode(), ctypes.byref(buf))
    out = json.loads(_take(buf)) if buf.value else {}
    if rc != 0:
        raise KeyError(name)
    return out["model"]


def tokenizer_encode(text: str | bytes, tokenizer_path: str | None = None) -> dict:
    """ids / pre-tokenizer pieces of `text` under a tokenizer.json (None = synthetic vocabulary)."""
    raw = text.encode() if isinstance(text, str) else text
    buf = ctypes.c_void_p()
    l = lib()
    l.acp_host_tokenizer_encode.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p)]
    rc = l.acp_host_tokenizer_encode(tokenizer_path.encode() if tokenizer_path else None, raw, len(raw), ctypes.byref(buf))
    out = json.loads(_take(buf)) if buf.value else {}
    if rc != 0:
        raise ValueError(out.get("error", f"acp_host_tokenizer_encode failed with {rc}"))
    return out


def tokenizer_decode(ids: list[int], tokenizer_path: str | None = None) -> bytes:
    arr = (ctypes.c_int * len(ids))(*ids)
    buf, n = ctypes.c_void_p(), ctypes.c_size_t()
    l = lib()
    l.acp_host_tokenizer_decode.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_int), ctypes.c_int,
                                            ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_size_t)]
    _check(l.acp_host_tokenizer_decode(tokenizer_path.encode() if tokenizer_path else None, arr, len(ids),
                                       ctypes.byref(buf), ctypes.byref(n)), "acp_host_tokenizer_decode")
    return _take(buf, n.value)


def render_prompt_with(request: dict, tokenizer_path: str | None) -> dict:
    raw = json.dumps(request).encode()
    buf = ctypes.c_void_p()
    l = lib()
    l.acp_host_render_prompt_with.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p)]
    rc = l.acp_host_render_prompt_with(tokenizer_path.encode() if tokenizer_path else None, raw, len(raw), ctypes.byref(buf))
    out = json.loads(_take(buf)) if buf.value else {}
    if rc != 0:
        raise ValueError(out.get("error", f"acp_host_render_prompt_with failed with {rc}"))
    return out


def checkpoint_tensor_bf16(path: str, name: str):
    """bf16 bit patterns (numpy uint16) of one checkpoint tensor as the loader would upload it."""
    import numpy as np
    l = lib()
    l.acp_host_checkpoint_tensor_bf16.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_size_t,
                                                  ctypes.POINTER(ctypes.c_size_t)]
    n = ctypes.c_size_t()
    _check(l.acp_host_checkpoint_tensor_bf16(path.encode(), name.encode(), None, 0, ctypes.byref(n)), "acp_host_checkpoint_tensor_bf16")
    out = np.empty(n.value, dtype=np.uint16)
    _check(l.acp_host_checkpoint_tensor_bf16(path.encode(), name.encode(), out.ctypes.data_as(ctypes.c_void_p), n.value,
                                             ctypes.byref(n)), "acp_host_checkpoint_tensor_bf16")
    return out

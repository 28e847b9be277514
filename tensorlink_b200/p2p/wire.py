"""The reference's wire format for shard calls, so that an H100 stage can sit behind an unmodified reference peer
(SURVEY.md §8 f-4).  Payload level only: sockets, packet prefixes and the DHT stay on the reference side.

Frame (what `tensor_to_bytes` / `bytes_to_tensor` exchange, /root/reference/tensorlink/ml/utils.py:569-660):

    [4-byte big-endian length n][n bytes of JSON skeleton][safetensors blob]

The skeleton is the payload with each tensor replaced by ``{"__tensor_ref__": "__tensor_<i>__", "dtype": "torch.bfloat16",
"shape": [...]}`` (i counts tensors in traversal order), each tuple by ``{"__tuple__": true, "data": [...]}``, scalars as
they are and anything else ``null``; the blob holds the tensors under those names.

Forward request (ml/module.py:1549-1556 -> ml/worker.py:301-307): ``[8-byte big-endian len(args frame)][args frame]
[kwargs frame]``; the reply is one frame holding the shard's output dict (ml/worker.py:344-346).

A ``DynamicCache`` is encoded like the reference does (``{"__dynamic_cache__": true, "key_cache": [...],
"value_cache": [...]}``, utils.py:599-605); ``decode`` leaves it as that dict (re-encoding it reproduces the same
bytes), because the stage keeps its KV cache resident and only inspects the shipped one for its length.

On-box hops never use this (they are device-to-device, p2p/link.py, p2p/peer.py); it exists for the boundary to the
reference's own processes.  tests/test_wire_cpu.py pins `encode` byte-for-byte to frames the reference produced.
"""
from __future__ import annotations

import json
from typing import Any, Dict, Tuple

import torch
from safetensors.torch import load as _blob_load
from safetensors.torch import save as _blob_save

_PLAIN = (int, float, bool, str, type(None))


def _is_dynamic_cache(node: Any) -> bool:
    return node.__class__.__name__ == "DynamicCache"


def _cache_lists(cache: Any):
    """Per-layer key / value tensors of an HF DynamicCache: ``key_cache`` / ``value_cache`` (transformers 4.x, what the
    reference reads, utils.py:600-603) or ``layers[i].keys`` / ``.values`` (5.x)."""
    if hasattr(cache, "key_cache"):
        return list(cache.key_cache), list(cache.value_cache)
    layers = getattr(cache, "layers", [])
    return ([getattr(l, "keys", None) for l in layers if getattr(l, "keys", None) is not None],
            [getattr(l, "values", None) for l in layers if getattr(l, "values", None) is not None])


class _Encoder:
    def __init__(self):
        self.tensors: Dict[str, torch.Tensor] = {}

    def walk(self, node: Any):
        if isinstance(node, torch.Tensor):
            name = "__tensor_%d__" % len(self.tensors)
            self.tensors[name] = node.detach().to("cpu").contiguous()
            return {"__tensor_ref__": name, "dtype": str(node.dtype), "shape": list(node.shape)}
        if isinstance(node, dict):
            return {key: self.walk(val) for key, val in node.items()}
        if _is_dynamic_cache(node):
            # utils.py:599-605: a DynamicCache travels as its per-layer key / value lists
            keys, vals = _cache_lists(node)
            return {"__dynamic_cache__": True, "key_cache": [self.walk(k) for k in keys],
                    "value_cache": [self.walk(v) for v in vals]}
        if isinstance(node, tuple):
            return {"__tuple__": True, "data": [self.walk(val) for val in node]}
        if isinstance(node, list):
            return [self.walk(val) for val in node]
        return node if isinstance(node, _PLAIN) else None


def encode(payload: Any) -> bytes:
    enc = _Encoder()
    head = json.dumps(enc.walk(payload)).encode("utf-8")
    blob = _blob_save(enc.tensors) if enc.tensors else b""
    return len(head).to_bytes(4, "big") + head + blob


def decode(frame: bytes, device=None) -> Any:
    """Inverse of ``encode``; tensors land on ``device`` when given."""
    if len(frame) < 4:
        raise ValueError("wire frame shorter than its length prefix")
    n = int.from_bytes(frame[:4], "big")
    if 4 + n > len(frame):
        raise ValueError(f"wire frame truncated: skeleton of {n} bytes in a frame of {len(frame)}")
    skeleton = json.loads(frame[4:4 + n].decode("utf-8"))
    blob = frame[4 + n:]
    tensors = _blob_load(bytes(blob)) if len(blob) else {}

    def build(node: Any):
        if isinstance(node, dict):
            ref = node.get("__tensor_ref__")
            if ref is not None:
                t = tensors[ref].to(dtype=getattr(torch, node["dtype"].split(".")[-1]))
                return t.to(device) if device is not None else t
            if node.get("__tuple__"):
                return tuple(build(v) for v in node["data"])
            return {k: build(v) for k, v in node.items()}
        if isinstance(node, list):
            return [build(v) for v in node]
        return node

    return build(skeleton)


def pack_forward(args: Any, kwargs: dict) -> bytes:
    a = encode(args)
    return len(a).to_bytes(8, "big") + a + encode(kwargs)


def unpack_forward(data: bytes, device=None) -> Tuple[Any, dict]:
    if len(data) < 8:
        raise ValueError("forward request shorter than its length prefix")
    n = int.from_bytes(data[:8], "big")
    if 8 + n > len(data):
        raise ValueError("forward request truncated")
    return decode(data[8:8 + n], device), decode(data[8 + n:], device)

"""``Torchnode``-shaped packet adapter: an H100 stage behind the reference's FORWARD / BACKWARD packets (SURVEY.md §8 f-4).

What the reference's network process does for the hot path (/root/reference/tensorlink/p2p/torch_node.py):

  user  -> worker   ``send_forward``   :825-836   b"FORWARD" + str(len(payload)) + b"::" + payload + json({"module_id", "key"})
                                                   payload = [8-byte len][args frame][kwargs frame]      (ml/module.py:1549-1556)
  worker: ``_handle_forward`` :251-299 parses it (``find(b"::")``, slice, JSON tail), copies the payload into shared memory
          and queues it under ``key``; the ML process polls, runs the shard, stores ``pickle.dumps(output frame)`` in shared
          memory (ml/worker.py:344-346, nodes/shared_memory.py:23-38 ``encoded=False``) and the node sends it back with
          ``send_forward`` under the same key (:524-530);
  user  -> worker   ``send_backward``  :865-869   b"BACKWARD" + str(len) + b"::" + gradient frame + json([n_batch, n_micro, module_id])
  worker -> user    the same packet shape carrying the input-gradient frame (ml/worker.py:289-291, raw frame: ``encoded=True``).

``B200Torchnode.handle_data(packet)`` takes such a packet as the reference's ``Connection`` delivers it (after its
EOT marker has been stripped, p2p/connection.py:67) and returns the reply packet the reference's user side expects —
no shared memory, no queues, no polling in between: the payload goes straight to ``DistributedWorker`` on the device.
Sockets, the RSA handshake and the DHT stay on the reference side (out of scope, SURVEY.md §2.1): this object is what
a reference ``Worker`` process would call instead of ``_store_tensor_in_shared_memory``.
"""
from __future__ import annotations

import json
import pickle
from typing import Optional, Tuple

EOT = b"HELLOCHENQUI"                       # p2p/connection.py:67: end-of-transmission marker of the reference's framing
MSG_FORWARD, MSG_BACKWARD = b"FORWARD", b"BACKWARD"


def build_forward(payload: bytes, key, module_id: str) -> bytes:
    """``Torchnode.send_forward`` (:825-836), byte for byte."""
    tail = json.dumps({"module_id": module_id, "key": key}).encode()
    return MSG_FORWARD + str(len(payload)).encode() + b"::" + payload + tail


def build_backward(payload: bytes, tag) -> bytes:
    """``Torchnode.send_backward`` (:865-869), byte for byte."""
    return MSG_BACKWARD + str(len(payload)).encode() + b"::" + payload + json.dumps(tag).encode()


def parse_forward(data: bytes) -> Tuple[bytes, Optional[str], tuple]:
    """``Torchnode._handle_forward`` (:251-299): (payload, module_id, key)."""
    if not data.startswith(MSG_FORWARD):
        raise ValueError("not a FORWARD packet")
    eos = data.find(b"::")
    if eos < 0:
        raise ValueError("FORWARD packet without a size field")
    size = int(data[len(MSG_FORWARD):eos])
    payload = data[eos + 2:eos + 2 + size]
    if len(payload) != size:
        raise ValueError(f"FORWARD packet truncated: {len(payload)} of {size} payload bytes")
    tail = json.loads(data[eos + 2 + size:])
    if isinstance(tail, dict):
        module_id, key = tail.get("module_id"), tail.get("key")
    else:
        module_id, key = None, tail
    return payload, module_id, tuple(key) if not isinstance(key, str) else key


def parse_backward(data: bytes) -> Tuple[bytes, tuple]:
    """``Torchnode._handle_backward`` (:225-249): (gradient frame, tag)."""
    if not data.startswith(MSG_BACKWARD):
        raise ValueError("not a BACKWARD packet")
    eos = data.find(b"::")
    if eos < 0:
        raise ValueError("BACKWARD packet without a size field")
    size = int(data[len(MSG_BACKWARD):eos])
    payload = data[eos + 2:eos + 2 + size]
    if len(payload) != size:
        raise ValueError(f"BACKWARD packet truncated: {len(payload)} of {size} payload bytes")
    return payload, tuple(json.loads(data[eos + 2 + size:]))


class B200Torchnode:
    """Packet front of one ``DistributedWorker`` (any object with ``handle_forward_frame`` / ``handle_backward_frame``)."""

    def __init__(self, worker):
        self.worker = worker
        self.ghosts = 0                      # packets for modules this node does not host (:253-255 counts them per peer)

    def handle_data(self, data: bytes) -> Optional[bytes]:
        """One received packet (EOT already stripped) -> the packet to send back, or None for an unknown packet type
        (the reference's dispatcher ignores those too)."""
        if data.endswith(EOT):
            data = data[:-len(EOT)]
        if data.startswith(MSG_FORWARD):
            payload, module_id, key = parse_forward(data)
            if module_id is None and not isinstance(key, str):
                module_id = key[2]                                   # (n_batch, n_micro, module_id): :838-851
            if module_id not in self.worker.modules:
                self.ghosts += 1
                raise KeyError(f"Unknown module_id in forward: {module_id}")          # the reference logs and drops (:280-284)
            frame = self.worker.handle_forward_frame(module_id, key, payload)
            # the reference's worker stores its reply with pickle (ml/worker.py:346 -> shared_memory.py:24-25)
            return build_forward(pickle.dumps(frame), list(key), module_id)
        if data.startswith(MSG_BACKWARD):
            payload, tag = parse_backward(data)
            module_id = tag[2]
            if module_id not in self.worker.modules:
                self.ghosts += 1
                raise KeyError(f"Unknown module_id in backward: {module_id}")
            return build_backward(self.worker.handle_backward_frame(module_id, tag, payload), list(tag))
        return None

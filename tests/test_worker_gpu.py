"""DistributedWorker mirror (tensorlink/ml/worker.py handler surface) over the CUDA stage."""
import pytest
import torch

from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml.weights import synthetic_tokens

pytestmark = pytest.mark.gpu


def test_two_workers_compose_like_one_shard_and_generate():
    from tensorlink_b200.ml import DistributedModel
    from tensorlink_b200.ml.worker import DistributedWorker
    cfg = C.TINY_QWEN2_D128
    w = DistributedWorker(max_batch=2, max_seq=64)
    a = w.load_module({"module_id": "a" * 64, "name": cfg.name, "type": "offloaded_group", "layer_range": (0, 1), "training": False})
    b = w.load_module({"module_id": "b" * 64, "name": cfg.name, "type": "offloaded_group", "layer_range": (2, 3), "training": False})
    full = w.load_module({"module_id": "f" * 64, "name": cfg.name, "type": "offloaded", "has_embed": True, "has_head": True})
    ids = synthetic_tokens(cfg, 2, 17).cuda()
    x0 = w.modules[full].embed(ids)
    o1 = w._handle_forward(a, (0, 0, a), {"hidden_states": x0, "use_cache": False, "position_ids": None})
    assert set(o1) == {"hidden_states", "use_cache", "position_ids"}           # kwargs ∪ outputs
    o2 = w._handle_forward(b, (0, 0, b), o1)
    ref = w._handle_forward(full, (0, 0, full), {"hidden_states": x0})
    assert torch.equal(o2["hidden_states"], ref["hidden_states"])              # sharded == unsharded, bit for bit

    class S:
        def __init__(self):
            self.cols, self.ended = [], False

        def put(self, t):
            self.cols.append(t)

        def end(self):
            self.ended = True
    s = S()
    got = w._handle_generate(full, ids, max_new_tokens=10, stream=s)
    want = DistributedModel(cfg, training=False, max_batch=2, max_seq=64).generate(ids, max_new_tokens=10)
    assert torch.equal(got, want)
    assert s.ended and torch.equal(torch.stack(s.cols, 1).cuda(), got[:, 17:])


def test_worker_training_ops():
    from tensorlink_b200.ml.worker import DistributedWorker
    cfg = C.TINY_QWEN2
    w = DistributedWorker(max_batch=2, max_seq=32)
    mid = w.load_module({"module_id": "t" * 64, "name": cfg.name, "type": "offloaded_group", "layer_range": (0, 3),
                         "training": True, "optimizer_type": "adam"})
    assert w.process_state_update(mid, ("init", {"lr": 1e-2})) == "loaded"
    assert w.process_state_update(mid, ("zero_grad", None)) == "zeroed"
    x = (torch.randn(2, 16, cfg.hidden, device="cuda") * 0.05).bfloat16()
    key = (0, 0, mid)
    y = w._handle_forward(mid, key, {"hidden_states": x})["hidden_states"]
    dx = w._handle_backward(mid, key, torch.randn_like(y) * 0.01)
    assert dx.shape == x.shape and torch.isfinite(dx.float()).all() and float(dx.float().abs().sum()) > 0
    before = w.modules[mid].params.flat.clone()
    assert w.process_state_update(mid, ("step", None)) == "stepped"
    assert float((w.modules[mid].params.flat.float() - before.float()).abs().sum()) > 0
    with pytest.raises(KeyError):
        w._handle_backward(mid, key, torch.randn_like(y))                      # intermediates are consumed once
    # the same backward framed as the reference frames it: identical input gradient
    from oracle import wire_oracle as W
    g = (torch.randn(2, 16, cfg.hidden) * 0.01).bfloat16()
    k1, k2 = (1, 0, mid), (1, 1, mid)
    w._handle_forward(mid, k1, {"hidden_states": x})
    w._handle_forward(mid, k2, {"hidden_states": x})
    direct = w._handle_backward(mid, k1, g.cuda())
    framed = W.decode(w.handle_backward_frame(mid, list(k2), W.encode(g)))
    assert framed.dtype == torch.bfloat16 and torch.equal(framed, direct.cpu())


def test_forward_in_the_reference_wire_format():
    """A forward request framed exactly as the reference user side frames it (8-byte length, args frame, kwargs frame with
    the loop live-ins) goes through ``handle_forward_frame`` and comes back as one frame whose hidden_states equal the
    direct call, with the other live-ins echoed like ``LayerGroupModule`` does."""
    from oracle import wire_oracle as W          # the reference-side encoder / decoder (test infrastructure)
    from tensorlink_b200.ml.worker import DistributedWorker
    cfg = C.TINY_QWEN2_D128
    w = DistributedWorker(max_batch=2, max_seq=64)
    a = w.load_module({"module_id": "a" * 64, "name": cfg.name, "type": "offloaded_group", "layer_range": (1, 2), "training": False})
    x = (torch.randn(2, 9, cfg.hidden) * 0.5).bfloat16()
    live_ins = {"hidden_states": x, "position_ids": torch.arange(9)[None].expand(2, -1).contiguous(), "use_cache": False,
                "causal_mask": None, "position_embeddings": (torch.zeros(2, 9, 8).bfloat16(), torch.ones(2, 9, 8).bfloat16())}
    args_frame, kwargs_frame = W.encode(()), W.encode(live_ins)
    request = len(args_frame).to_bytes(8, "big") + args_frame + kwargs_frame
    reply = W.decode(w.handle_forward_frame(a, (0, 0, a), request))
    direct = w._handle_forward(a, (0, 1, a), {"hidden_states": x.cuda()})
    assert set(reply) == set(live_ins)
    assert reply["hidden_states"].dtype == torch.bfloat16 and torch.equal(reply["hidden_states"], direct["hidden_states"].cpu())
    assert torch.equal(reply["position_ids"], live_ins["position_ids"]) and reply["use_cache"] is False
    assert isinstance(reply["position_embeddings"], tuple) and torch.equal(reply["position_embeddings"][1], live_ins["position_embeddings"][1])
    with pytest.raises(KeyError):
        w.handle_forward_frame(a, (0, 2, a), (len(args_frame)).to_bytes(8, "big") + args_frame + W.encode({"use_cache": True}))


def test_cached_decode_call_from_a_reference_peer():
    """What an unmodified reference user ships for a cached decode step (injector.py:508-556): hidden_states [B,1,H],
    ``cache_position`` / ``position_ids`` naming the position and the whole DynamicCache.  The stage's KV cache is
    resident: the position comes from the live-ins, is checked against the resident cache, and the step equals the
    direct cached call; inputs the executor cannot honour raise instead of computing at position 0."""
    from oracle import wire_oracle as W
    from tensorlink_b200.ml.worker import DistributedWorker
    cfg = C.TINY_QWEN2_D128
    w = DistributedWorker(max_batch=1, max_seq=64)
    a = w.load_module({"module_id": "a" * 64, "name": cfg.name, "type": "offloaded_group", "layer_range": (0, 1), "training": False})
    b = w.load_module({"module_id": "b" * 64, "name": cfg.name, "type": "offloaded_group", "layer_range": (0, 1), "training": False})
    x = (torch.randn(1, 7, cfg.hidden) * 0.5).bfloat16()
    x1 = (torch.randn(1, 1, cfg.hidden) * 0.5).bfloat16()
    # module b: the direct cached call (prefill 7, then one token at past_len 7)
    w._handle_forward(b, (0, 0, b), {"hidden_states": x.cuda()})
    want = w._handle_forward(b, (1, 0, b), {"hidden_states": x1.cuda(), "past_len": 7})["hidden_states"].cpu()
    # module a: the same two calls framed like the reference frames them
    def req(kw):
        af = W.encode(())
        return len(af).to_bytes(8, "big") + af + W.encode(kw)
    w.handle_forward_frame(a, (0, 0, a), req({"hidden_states": x, "cache_position": torch.arange(7), "use_cache": True}))

    class DynamicCache:                         # transformers-4.x attribute names, what the reference codec reads
        def __init__(self, k, v):
            self.key_cache, self.value_cache = k, v
    shipped = DynamicCache([torch.zeros(1, cfg.n_kv_heads, 7, cfg.head_dim).bfloat16()] * 2,
                           [torch.zeros(1, cfg.n_kv_heads, 7, cfg.head_dim).bfloat16()] * 2)
    step = {"hidden_states": x1, "cache_position": torch.tensor([7]), "position_ids": torch.tensor([[7]]), "use_cache": True,
            "past_key_values": shipped}
    got = W.decode(w.handle_forward_frame(a, (1, 0, a), req(step)))
    assert torch.equal(got["hidden_states"], want)
    assert got["past_key_values"]["__dynamic_cache__"] is True            # echoed like LayerGroupModule echoes its kwargs
    # a call whose position disagrees with the resident cache, or with padding, must not run silently
    with pytest.raises(ValueError):
        w.handle_forward_frame(a, (2, 0, a), req({"hidden_states": x1, "cache_position": torch.tensor([3])}))
    with pytest.raises(NotImplementedError):
        w.handle_forward_frame(a, (3, 0, a), req({"hidden_states": x, "attention_mask": torch.tensor([[0, 0, 1, 1, 1, 1, 1]])}))
    with pytest.raises(NotImplementedError):
        w.handle_forward_frame(a, (4, 0, a), req({"hidden_states": x, "position_ids": torch.tensor([[0, 0, 0, 1, 2, 3, 4]])}))


def test_generate_bounds_are_checked():
    from tensorlink_b200.ml.worker import DistributedWorker
    cfg = C.TINY_QWEN2
    w = DistributedWorker(max_batch=1, max_seq=32)
    full = w.load_module({"module_id": "f" * 64, "name": cfg.name, "type": "offloaded", "has_embed": True, "has_head": True})
    with pytest.raises(ValueError):
        w._handle_generate(full, synthetic_tokens(cfg, 1, 30).cuda(), max_new_tokens=8)      # 38 > max_seq: would write past the cache
    with pytest.raises(ValueError):
        w._handle_generate(full, synthetic_tokens(cfg, 2, 8).cuda(), max_new_tokens=4)       # 2 rows > max_batch


def test_forward_and_backward_packets_through_the_torchnode_adapter():
    """The reference's FORWARD / BACKWARD packets (p2p/torch_node.py:825-836, :865-869) in, reply packets out, over a real
    stage: what a reference user process would exchange with an H100 worker (SURVEY.md §8 f-4)."""
    import pickle
    from oracle import wire_oracle as W
    from tensorlink_b200.ml.worker import DistributedWorker
    from tensorlink_b200.p2p import torch_node as T
    cfg = C.TINY_QWEN2
    w = DistributedWorker(max_batch=2, max_seq=32)
    mid = w.load_module({"module_id": "c" * 64, "name": cfg.name, "type": "offloaded_group", "layer_range": (0, 1), "training": True})
    node = T.B200Torchnode(w)
    x = (torch.randn(2, 8, cfg.hidden) * 0.1).bfloat16()
    key = [0, 0, mid]
    af = W.encode(())
    request = T.build_forward(len(af).to_bytes(8, "big") + af + W.encode({"hidden_states": x, "use_cache": False}), key, mid)
    reply = node.handle_data(request)
    payload, module_id, rkey = T.parse_forward(reply)
    out = W.decode(pickle.loads(payload))                                  # the reference user unpickles, then decodes the frame
    assert module_id == mid and rkey == tuple(key) and out["use_cache"] is False
    direct = w._handle_forward(mid, (9, 9, mid), {"hidden_states": x.cuda()})["hidden_states"].cpu()
    assert torch.equal(out["hidden_states"], direct)
    g = (torch.randn(2, 8, cfg.hidden) * 0.01).bfloat16()
    back = node.handle_data(T.build_backward(W.encode(g), key))
    gframe, tag = T.parse_backward(back)
    want = w._handle_backward(mid, (9, 9, mid), g.cuda()).cpu()
    assert tag == tuple(key) and torch.equal(W.decode(gframe), want)

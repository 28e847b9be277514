"""Qwen3-MoE on the CPU: the MoE oracle against HF's Qwen3MoeForCausalLM (eager attention and experts), parameter counts,
config parsing and what raises, checkpoint round trips in both of HF's expert layouts, and stage placement."""
import json

import pytest
import torch

from oracle import shard_oracle as O
from tensorlink_b200.ml import configs as C
from tensorlink_b200.ml import graphing
from tensorlink_b200.ml.checkpoint import LazyCheckpoint, config_from_dir, config_to_json, save_checkpoint
from tensorlink_b200.ml.module import _config_from_hf
from tensorlink_b200.ml.shard import ShardParams
from tensorlink_b200.ml.weights import init_state_dict, synthetic_tokens
from tests.moe_oracle import MoeOracleModel, hf_model

CASES = [C.TINY_QWEN3_MOE, C.TINY_QWEN3_MOE_UNNORM]
MOE_KEYS = ("hidden", "intermediate", "n_layers", "n_heads", "n_kv_heads", "head_dim", "vocab", "tied", "qkv_bias", "qk_norm",
            "rope_theta", "rms_eps", "max_pos", "n_experts", "top_k", "moe_intermediate", "norm_topk_prob")


def _same_cfg(a, b):
    return all(getattr(a, k) == getattr(b, k) for k in MOE_KEYS)


def test_param_counts():
    c = C.QWEN3_30B_A3B
    assert c.total_params() == 30_532_122_624
    assert c.active_params() == 3_353_032_704
    assert C.QWEN3_8B.active_params() == C.QWEN3_8B.total_params()
    assert 2 * c.total_params() / 1e9 == pytest.approx(61.06, abs=0.01)


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
def test_oracle_bit_exact_vs_hf(cfg):
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 2, 24)
    hf = hf_model(cfg, sd)
    with torch.no_grad():
        ref = hf(input_ids=ids).logits
        got = MoeOracleModel(cfg, sd, "eager").logits(ids)
        got3 = MoeOracleModel(cfg, sd, "eager").logits(ids, n_shards=3)
    assert torch.equal(got, ref)
    assert torch.equal(got3, ref)            # sharded == unsharded


@pytest.mark.parametrize("cfg", CASES, ids=lambda c: c.name)
def test_oracle_greedy_ids_equal_hf_generate(cfg):
    sd = init_state_dict(cfg)
    ids = synthetic_tokens(cfg, 1, 12)
    hf = hf_model(cfg, sd)
    with torch.no_grad():
        ref = hf.generate(ids, max_new_tokens=8, do_sample=False, pad_token_id=0, eos_token_id=None)
    got = MoeOracleModel(cfg, sd, "eager").generate(ids, 8)
    assert torch.equal(got, ref)


def test_config_from_hf_module_and_config_json(tmp_path):
    cfg = C.TINY_QWEN3_MOE_UNNORM
    sd = init_state_dict(cfg)
    m = hf_model(cfg, sd)
    assert _same_cfg(_config_from_hf(m), cfg)
    with open(tmp_path / "config.json", "w") as f:
        json.dump(config_to_json(cfg), f)
    assert _same_cfg(config_from_dir(str(tmp_path)), cfg)


def _write_config(path, **over):
    c = config_to_json(C.TINY_QWEN3_MOE)
    c.update(over)
    with open(path / "config.json", "w") as f:
        json.dump(c, f)


@pytest.mark.parametrize("over, what", [
    ({"model_type": "qwen2_moe", "shared_expert_intermediate_size": 256}, "qwen3_moe"),
    ({"mlp_only_layers": [1]}, "mixed dense and sparse"),
    ({"decoder_sparse_step": 2}, "mixed dense and sparse"),
    ({"quantization_config": {"quant_method": "fp8", "fmt": "e4m3", "weight_block_size": [128, 128],
                              "activation_scheme": "dynamic"}}, "FP8"),
    ({"num_experts": 512}, "experts"),
    ({"num_experts_per_tok": 17}, "top_k"),
])
def test_unsupported_configs_raise(tmp_path, over, what):
    from tensorlink_b200.ml import DistributedModel
    _write_config(tmp_path, **over)
    with pytest.raises(NotImplementedError, match=what):
        DistributedModel(str(tmp_path), training=False)


def test_training_and_router_logits_raise():
    from tensorlink_b200.ml import DistributedModel
    with pytest.raises(NotImplementedError, match="training"):
        DistributedModel(C.TINY_QWEN3_MOE, training=True)
    with pytest.raises(NotImplementedError, match="FP8"):
        ShardParams(C.TINY_QWEN3_MOE, [0], False, False, "cpu", fp8=True)
    m = hf_model(C.TINY_QWEN3_MOE, init_state_dict(C.TINY_QWEN3_MOE))
    m.config.output_router_logits = True
    with pytest.raises(NotImplementedError, match="output_router_logits"):
        _config_from_hf(m)


def _arena(cfg, sd):
    p = ShardParams(cfg, range(cfg.n_layers), True, True, "cpu")
    p.load_hf_state_dict(sd)
    return p


def test_hf_save_pretrained_loads_into_the_same_arena(tmp_path):
    cfg = C.TINY_QWEN3_MOE
    sd = init_state_dict(cfg)
    hf_model(cfg, sd).save_pretrained(tmp_path)
    ck = LazyCheckpoint(str(tmp_path))
    assert "model.layers.0.mlp.experts.3.up_proj.weight" in ck          # transformers writes one tensor per expert
    assert _same_cfg(config_from_dir(str(tmp_path)), cfg)
    want = _arena(cfg, sd)
    got = _arena(cfg, ck)
    assert torch.equal(got.flat, want.flat)
    out = want.hf_state_dict()                                           # fused names, like model.state_dict()
    assert set(out) == set(sd) and all(torch.equal(out[k], sd[k]) for k in sd)


class _Link:
    rank, world = 0, 1

    def all_gather_object(self, o):
        return [o]

    def barrier(self):
        pass


def test_project_writer_loads_in_transformers(tmp_path):
    from transformers import AutoModelForCausalLM
    cfg = C.TINY_QWEN3_MOE_UNNORM
    sd = init_state_dict(cfg)

    class _DM:
        pass
    dm = _DM()
    dm.cfg, dm.stage = cfg, _DM()
    dm.stage.params = _arena(cfg, sd)
    save_checkpoint(dm, str(tmp_path), link=_Link())
    ck = LazyCheckpoint(str(tmp_path))
    assert "model.layers.2.mlp.experts.31.down_proj.weight" in ck and "model.layers.2.mlp.experts.down_proj" not in ck
    m = AutoModelForCausalLM.from_pretrained(str(tmp_path), dtype=torch.bfloat16, attn_implementation="eager",
                                             experts_implementation="eager").eval()
    ids = synthetic_tokens(cfg, 2, 16)
    with torch.no_grad():
        ref = MoeOracleModel(cfg, sd, "eager").logits(ids)
        got = m(input_ids=ids).logits
    assert torch.equal(got, ref)


def test_stages_hold_about_equal_parameters():
    cfg = C.QWEN3_30B_A3B
    for n in (2, 3, 4):
        parts = graphing.split_balanced(cfg, n)
        assert [i for r in parts for i in r] == list(range(cfg.n_layers))
        sizes = [len(r) * cfg.layer_params() + (cfg.vocab * cfg.hidden if i in (0, n - 1) else 0) for i, r in enumerate(parts)]
        assert max(sizes) / min(sizes) < 1.1, sizes
        plan = graphing.make_plan(cfg, n, balanced=True)
        assert graphing.n_stages(plan) == n


@pytest.mark.parametrize("model_type, extra", [("mixtral", {"num_local_experts": 8}), ("deepseek_v3", {"n_routed_experts": 256}),
                                               ("dbrx", {"ffn_config": {"moe_num_experts": 16}})])
def test_other_moe_families_from_hf_modules_raise(model_type, extra):
    from types import SimpleNamespace
    c = SimpleNamespace(model_type=model_type, hidden_size=512, intermediate_size=1024, num_hidden_layers=2,
                        num_attention_heads=4, num_key_value_heads=2, vocab_size=2048, tie_word_embeddings=False,
                        rms_norm_eps=1e-6, max_position_embeddings=4096, **extra)
    with pytest.raises(NotImplementedError, match="qwen3_moe"):
        _config_from_hf(SimpleNamespace(config=c))

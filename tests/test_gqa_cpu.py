"""Grouped-query attention (num_key_value_heads < num_attention_heads) without a GPU: the oracle's `repeat_kv` restatement is pinned to
the reference layer's own GQA outputs (tests/golden/gqa_*.npz, oracle/gen_golden_gqa.py), the layer's parameters match the reference's,
unsupported head counts are refused, and both gradient-bucket planners keep the narrower q|k|v row blocks in one bucket."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import decoder_oracle as O
from oracle import gqa_oracle as G
from oracle import gen_golden, gen_golden_gqa

GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")
LAYERS = sorted(glob.glob(os.path.join(GOLDEN_DIR, "gqa_layer_*.npz")))
BF = torch.bfloat16


def _bf16(bits):
    return torch.from_numpy(bits.view(np.int16)).view(BF)


def test_gqa_goldens_present():
    names = {os.path.basename(p) for p in LAYERS}
    assert names == {f"gqa_layer_{n}.npz" for n in gen_golden_gqa.CASES}
    for p in LAYERS + [os.path.join(GOLDEN_DIR, f) for f in ("gqa_kvcache_layer.npz", "gqa_bf16_pins.npz")]:
        assert os.path.getsize(p) < 1 << 20, p


@pytest.mark.parametrize("path", LAYERS, ids=[os.path.basename(p) for p in LAYERS])
def test_oracle_matches_reference_gqa_golden(path):
    g = np.load(path)
    hidden, inter, heads, bsz, seq, seed, pad = [int(v) for v in g["shape"]]
    kv_heads, theta = int(g["kv_heads"]), float(g["rope_theta"])
    rs, cs = [int(v) for v in g["stride"]]
    p = {k: v.requires_grad_(True) for k, v in G.init_layer_params(hidden, inter, seed, heads, kv_heads).items()}
    x, gy = gen_golden.make_inputs(hidden, bsz, seq, seed)
    x.requires_grad_(True)
    am = gen_golden_gqa.pad_mask(bsz, seq, pad)
    valid = torch.ones(bsz, seq, dtype=torch.bool) if am is None else am.bool()
    if am is not None:
        gy = gy * am[..., None]
    assert gen_golden.checksum(x.detach()) == pytest.approx(float(g["x_checksum"]), rel=1e-12)
    assert sum(gen_golden.checksum(v.detach()) for v in p.values()) == pytest.approx(float(g["w_checksum"]), rel=1e-12)
    cos, sin = O.rope_tables(hidden // heads, 2048, base=theta)
    pos = torch.arange(seq)[None].expand(bsz, -1)
    y = G.decoder_layer(x, p, heads, kv_heads, cos, sin, pos, O.causal_additive_mask(bsz, seq, torch.float32, am))
    y.backward(gy)
    vs = valid[:, ::rs]
    np.testing.assert_allclose(y.detach()[:, ::rs, ::cs][vs].numpy(), g["y"][vs.numpy()], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(x.grad[:, ::rs, ::cs][vs].numpy(), g["dx"][vs.numpy()], rtol=1e-4, atol=1e-7)
    assert gen_golden.checksum(y.detach()[valid]) == pytest.approx(float(g["y_abs_sum"]), rel=1e-5)
    assert gen_golden.checksum(x.grad[valid]) == pytest.approx(float(g["dx_abs_sum"]), rel=1e-5)
    for k, v in p.items():
        gr = v.grad
        np.testing.assert_allclose((gr[:8, :64] if gr.dim() == 2 else gr).numpy(), g["d_" + k], rtol=1e-4, atol=1e-7, err_msg=k)
        assert float(gr.double().sum()) == pytest.approx(float(g["dsum_" + k]), rel=1e-3, abs=1e-6)


def test_kvcache_oracle_matches_reference_gqa_golden():
    g = np.load(os.path.join(GOLDEN_DIR, "gqa_kvcache_layer.npz"))
    hidden, inter, heads, kv_heads = [int(v) for v in g["shape"]]
    p, calls = G.cached_decode_scenario(hidden, inter, heads, kv_heads)
    outs = G.run_cached_scenario(p, calls, heads, kv_heads)
    assert len(outs) == 4
    for i, ((x, am, pos), y) in enumerate(zip(calls, outs)):
        assert np.array_equal(am.numpy(), g[f"mask{i}"])
        valid = am[:, -x.shape[1]:].bool()
        np.testing.assert_allclose(y.detach()[valid].numpy(), g[f"y{i}"][valid.numpy()], rtol=1e-5, atol=1e-6, err_msg=f"call {i}")


def test_oracle_matches_reference_gqa_bf16_pins():
    """bf16: the oracle's GQA path shares the reference's rounding points, bit for bit, for a causal forward and the kv-cache scenario."""
    g = np.load(os.path.join(GOLDEN_DIR, "gqa_bf16_pins.npz"))
    hidden, inter, heads, kv_heads, bsz, seq, seed = gen_golden_gqa.BF16_LAYER_CASE
    pb = {k: v.to(BF) for k, v in G.init_layer_params(hidden, inter, seed, heads, kv_heads).items()}
    x, _ = gen_golden.make_inputs(hidden, bsz, seq, seed)
    cos, sin = O.rope_tables(hidden // heads, 2048, dtype=BF)
    pos = torch.arange(seq)[None].expand(bsz, -1)
    y = G.decoder_layer(x.to(BF), pb, heads, kv_heads, cos, sin, pos, O.causal_additive_mask(bsz, seq, BF))
    assert torch.equal(y, _bf16(g["layer_y"]))
    hidden, inter, heads, kv_heads = gen_golden_gqa.KV_CASE
    p, calls = G.cached_decode_scenario(hidden, inter, heads, kv_heads)
    outs = G.run_cached_scenario(p, calls, heads, kv_heads, dtype=BF)
    for i, ((x, am, pos), y) in enumerate(zip(calls, outs)):
        valid = am[:, -x.shape[1]:].bool()
        assert torch.equal(_bf16(g[f"kv_y{i}"])[valid], y[valid]), f"call {i}"


def test_gqa_params_with_kv_heads_equal_heads_are_the_multi_head_params():
    """gqa_oracle draws decoder_oracle's RNG stream: with kv_heads == heads it gives exactly the multi-head parameters."""
    a = O.init_layer_params(256, 512, 11)
    b = G.init_layer_params(256, 512, 11, 2, 2)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize("path", LAYERS, ids=[os.path.basename(p) for p in LAYERS])
def test_gqa_layer_state_dict_matches_reference(path):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer
    g = np.load(path)
    hidden, inter, heads = [int(v) for v in g["shape"][:3]]
    layer = DreamLLMDecoderLayer(DreamLLMConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=heads,
                                                num_key_value_heads=int(g["kv_heads"]), rope_theta=float(g["rope_theta"])))
    ours = {k: list(v.shape) + [0] * (2 - v.dim()) for k, v in layer.state_dict().items()}
    want = {str(k): [int(s) for s in shp] for k, shp in zip(g["sd_names"], g["sd_shapes"])}
    assert ours == want


@pytest.mark.parametrize("heads,kv_heads", [(8, 3), (4, 8), (6, 4)])
def test_kv_heads_must_divide_heads(heads, kv_heads):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer, DreamLLMModel
    cfg = DreamLLMConfig(hidden_size=64 * heads, intermediate_size=256, num_attention_heads=heads, num_key_value_heads=kv_heads,
                         num_hidden_layers=1)
    with pytest.raises(ValueError, match="multiple of num_key_value_heads"):
        DreamLLMDecoderLayer(cfg)
    with pytest.raises(ValueError, match="multiple of num_key_value_heads"):
        DreamLLMModel(cfg)


def _gqa_params(kv_heads, layers=3):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=96, hidden_size=512, intermediate_size=640, num_hidden_layers=layers, num_attention_heads=8,
                         num_key_value_heads=kv_heads)
    m = DreamLLMForCausalMLM(cfg).to(BF)
    return m, list(m.parameters())


def _qkv_triples(m):
    return [(l.self_attn.q_proj.weight, l.self_attn.k_proj.weight, l.self_attn.v_proj.weight) for l in m.model.layers]


def _adjacent(bucket, triple):
    ids = [id(p) for p in bucket]
    at = [ids.index(id(p)) if id(p) in ids else -1 for p in triple]
    return at[0] >= 0 and at[1] == at[0] + 1 and at[2] == at[0] + 2


CAPS_MB = [0.0001, 0.05, 0.3, 0.5, 0.6, 0.75, 1.0, 1.5, 2.5, 4.0, 1e4]


@pytest.mark.parametrize("kv_heads", [2, 1, 4])
def test_reducer_plan_keeps_qkv_in_one_bucket(kv_heads):
    from dreamllm_b200.ddp import plan_buckets
    m, params = _gqa_params(kv_heads)
    for cap in CAPS_MB:
        plan = plan_buckets(params, int(cap * 1024 * 1024))
        assert sorted(id(p) for b in plan for p in b) == sorted(id(p) for p in params)
        for triple in _qkv_triples(m):
            assert sum(_adjacent(b, triple) for b in plan) == 1, (cap, [p.shape for p in triple])


@pytest.mark.parametrize("kv_heads", [2, 1, 4])
def test_sharded_adamw_keeps_qkv_in_one_bucket(kv_heads):
    from dreamllm_b200.modeling_dreamllm import _fuse_rows
    from dreamllm_b200.zero import ShardedAdamW
    from oracle import adamw_oracle as AO
    for cap in CAPS_MB:
        m, params = _gqa_params(kv_heads)
        opt = ShardedAdamW(params, lr=1e-3, bucket_cap_mb=cap, update_fn=AO.adamw_flat_, sumsq_fn=AO.sumsq_flat)
        for triple in _qkv_triples(m):
            assert sum(_adjacent(b.params, triple) for b in opt.buckets) == 1, (cap, [p.shape for p in triple])
            w = _fuse_rows(list(triple))                     # adjacent in the bucket: the fused weight is a view, not a re-allocation
            assert w.data_ptr() == triple[0].data_ptr() and w.shape[0] == sum(p.shape[0] for p in triple)

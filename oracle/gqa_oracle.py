"""TEST INFRASTRUCTURE ONLY — grouped-query attention (num_key_value_heads < num_attention_heads) for the CPU oracle.

The decoder layer of oracle/decoder_oracle.py with k_proj / v_proj of num_kv_heads * head_dim rows: keys / values are projected and
rotated at nkv heads, cached at nkv heads, and repeated to the query heads by `repeat_kv` right before the attention products (reference
modeling_dreamllm.py:242-252, :344-358).  Everything else (RMSNorm, RoPE, masks, MLP) is decoder_oracle's own code, so the rounding
points are the reference's.  With num_kv_heads == num_heads every function here computes what its decoder_oracle namesake does.

Pinned by tests/test_gqa_cpu.py against tests/golden/gqa_*.npz, minted by oracle/gen_golden_gqa.py from the reference's own layer.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import decoder_oracle as O


def repeat_kv(x, n_rep: int):
    """:242-252: [B, nkv, S, d] -> [B, nkv * n_rep, S, d], kv head j serving q heads j * n_rep .. j * n_rep + n_rep - 1."""
    if n_rep == 1:
        return x
    b, nkv, s, d = x.shape
    return x[:, :, None].expand(b, nkv, n_rep, s, d).reshape(b, nkv * n_rep, s, d)


def init_layer_params(hidden, inter, seed, heads, kv_heads, dtype=torch.float32, std=0.02):
    """decoder_oracle.init_layer_params with k_proj / v_proj of kv_heads * head_dim rows: the same RNG draws in the same order, so
    kv_heads == heads gives exactly the multi-head parameters."""
    g = torch.Generator().manual_seed(seed)
    kv_rows = kv_heads * (hidden // heads)
    shapes = {
        "self_attn.q_proj.weight": (hidden, hidden),
        "self_attn.k_proj.weight": (kv_rows, hidden),
        "self_attn.v_proj.weight": (kv_rows, hidden),
        "self_attn.o_proj.weight": (hidden, hidden),
        "mlp.gate_proj.weight": (inter, hidden),
        "mlp.up_proj.weight": (inter, hidden),
        "mlp.down_proj.weight": (hidden, inter),
    }
    p = {k: (torch.randn(s, generator=g) * std).to(dtype) for k, s in shapes.items()}
    p["input_layernorm.weight"] = (1.0 + 0.1 * torch.randn(hidden, generator=g)).to(dtype)
    p["post_attention_layernorm.weight"] = (1.0 + 0.1 * torch.randn(hidden, generator=g)).to(dtype)
    return p


def attention_eager(x, wq, wk, wv, wo, num_heads, num_kv_heads, cos, sin, position_ids, mask4d, past_kv=None, return_kv=False):
    """DreamLLMAttention.forward (eager path), :309-400, with nkv = num_kv_heads.  `past_kv` = (k, v) [B, nkv, past, d] already rotated;
    the present `(k, v)` keeps nkv heads (:355), `repeat_kv` comes after the cache update (:357-358)."""
    bsz, q_len, hidden = x.shape
    d = hidden // num_heads
    q = F.linear(x, wq).view(bsz, q_len, num_heads, d).transpose(1, 2)
    k = F.linear(x, wk).view(bsz, q_len, num_kv_heads, d).transpose(1, 2)
    v = F.linear(x, wv).view(bsz, q_len, num_kv_heads, d).transpose(1, 2)
    q, k = O.apply_rope(q, k, cos.to(x.dtype), sin.to(x.dtype), position_ids)
    if past_kv is not None:
        k = torch.cat([past_kv[0], k], dim=2)
        v = torch.cat([past_kv[1], v], dim=2)
    present = (k, v)
    k, v = repeat_kv(k, num_heads // num_kv_heads), repeat_kv(v, num_heads // num_kv_heads)
    w = torch.matmul(q, k.transpose(2, 3)) / math.sqrt(d)
    if mask4d is not None:
        w = w + mask4d
        w = torch.max(w, torch.tensor(torch.finfo(w.dtype).min, dtype=w.dtype))  # :373-375
    w = F.softmax(w, dim=-1, dtype=torch.float32).to(q.dtype)  # :378
    o = torch.matmul(w, v).transpose(1, 2).contiguous().reshape(bsz, q_len, hidden)
    out = F.linear(o, wo)
    return (out, present) if return_kv else out


def decoder_layer(x, p: dict, num_heads, num_kv_heads, cos, sin, position_ids, mask4d, eps=1e-6, past_kv=None, return_kv=False):
    """DreamLLMDecoderLayer.forward, :599-654, with grouped-query attention; `p` uses the reference's state-dict key names."""
    h = O.rmsnorm(x, p["input_layernorm.weight"], eps)
    h = attention_eager(h, p["self_attn.q_proj.weight"], p["self_attn.k_proj.weight"], p["self_attn.v_proj.weight"],
                        p["self_attn.o_proj.weight"], num_heads, num_kv_heads, cos, sin, position_ids, mask4d, past_kv=past_kv,
                        return_kv=return_kv)
    present = None
    if return_kv:
        h, present = h
    x = x + h
    h = O.mlp(O.rmsnorm(x, p["post_attention_layernorm.weight"], eps), p["mlp.gate_proj.weight"], p["mlp.up_proj.weight"],
              p["mlp.down_proj.weight"])
    return (x + h, present) if return_kv else x + h


def cached_decode_scenario(hidden, inter, heads, kv_heads, seed=21, lens=(37, 50), steps=3):
    """decoder_oracle.cached_decode_scenario (left-padded prompt batch, prefill + `steps` single-token steps, HF generate's masks and
    positions) with grouped-query parameters; the inputs are drawn exactly as there."""
    p = init_layer_params(hidden, inter, seed, heads, kv_heads)
    _, calls = O.cached_decode_scenario(hidden, inter, heads, seed, lens, steps)
    return p, calls


def run_cached_scenario(p, calls, heads, kv_heads, dtype=torch.float32):
    """Oracle outputs of `cached_decode_scenario`: list of hidden states [B, S_i, H] (pad rows included; compare valid rows only)."""
    pp = {k: v.to(dtype) for k, v in p.items()}
    d = calls[0][0].shape[-1] // heads
    cos, sin = O.rope_tables(d, 2048, dtype=dtype)
    past, outs = None, []
    for x, am, pos in calls:
        past_len = 0 if past is None else past[0].shape[2]
        mask = O.causal_additive_mask_past(x.shape[0], x.shape[1], past_len, dtype, am)
        y, past = decoder_layer(x.to(dtype), pp, heads, kv_heads, cos, sin, pos, mask, past_kv=past, return_kv=True)
        outs.append(y)
    return outs

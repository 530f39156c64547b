"""TEST INFRASTRUCTURE ONLY — the attention weights of the reference's eager path (`output_attentions=True`) for the CPU oracle.

DreamLLMAttention.forward returns the post-softmax probabilities [B, nh, q_len, kv_len] it multiplies V with (reference
modeling_dreamllm.py:357-378): repeat_kv, q k^T / sqrt(d) in the model dtype, additive 4-D mask, clamp to finfo.min (:373-375), softmax
in fp32, cast back to the model dtype.  This module restates exactly that on top of the unchanged decoder_oracle / gqa_oracle (their
RMSNorm, projections, RoPE, masks and kv-cache scenario), so the rounding points are the reference's.  What the clamp implies:

  * masked keys are exactly 0;
  * a right-padded query row (training-style 2-D mask) is NOT zero: the padding mask masks keys only, so it is a softmax over the
    sample's valid keys;
  * a row with no visible key (a left-padded prompt position, a length-0 sample) has every score equal to finfo.min: uniform 1/kv_len.

Pinned by tests/test_attn_weights_cpu.py against tests/golden/attn_weights_*.npz, minted by oracle/gen_golden_attn_weights.py from the
reference's own layer.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import decoder_oracle as O
from oracle import gqa_oracle as G


def core_weights(q, k, mask4d):
    """:357-378 from rotated q [B, nh, q_len, d] and k [B, nkv, kv_len, d] (past keys included): the weights in q's dtype."""
    nh, nkv, d = q.shape[1], k.shape[1], q.shape[-1]
    k = G.repeat_kv(k, nh // nkv)
    w = torch.matmul(q, k.transpose(2, 3)) / math.sqrt(d)
    if mask4d is not None:
        w = w + mask4d
        w = torch.max(w, torch.tensor(torch.finfo(w.dtype).min, dtype=w.dtype))
    return F.softmax(w, dim=-1, dtype=torch.float32).to(q.dtype)


def qk_states(x, p, num_heads, num_kv_heads, cos, sin, position_ids, eps=1e-6):
    """input_layernorm -> q_proj / k_proj -> RoPE of one decoder layer (:309-348): q [B, nh, S, d], k [B, nkv, S, d]."""
    bsz, q_len, hidden = x.shape
    d = hidden // num_heads
    h = O.rmsnorm(x, p["input_layernorm.weight"], eps)
    q = F.linear(h, p["self_attn.q_proj.weight"]).view(bsz, q_len, num_heads, d).transpose(1, 2)
    k = F.linear(h, p["self_attn.k_proj.weight"]).view(bsz, q_len, num_kv_heads, d).transpose(1, 2)
    return O.apply_rope(q, k, cos.to(x.dtype), sin.to(x.dtype), position_ids)


def layer_weights(x, p, num_heads, num_kv_heads, cos, sin, position_ids, mask4d, eps=1e-6, past_k=None):
    """DreamLLMDecoderLayer.forward(output_attentions=True)[1]; `past_k` [B, nkv, past, d] are the cached (rotated) keys."""
    q, k = qk_states(x, p, num_heads, num_kv_heads, cos, sin, position_ids, eps)
    if past_k is not None:
        k = torch.cat([past_k, k], dim=2)
    return core_weights(q, k, mask4d)


def run_cached_scenario(p, calls, heads, kv_heads, dtype=torch.float32):
    """Weights of every call of gqa_oracle.cached_decode_scenario (prefill + single-token steps): list of [B, nh, S_i, past_i + S_i]."""
    pp = {k: v.to(dtype) for k, v in p.items()}
    d = calls[0][0].shape[-1] // heads
    cos, sin = O.rope_tables(d, 2048, dtype=dtype)
    past, outs = None, []
    for x, am, pos in calls:
        past_len = 0 if past is None else past[0].shape[2]
        mask = O.causal_additive_mask_past(x.shape[0], x.shape[1], past_len, dtype, am)
        outs.append(layer_weights(x.to(dtype), pp, heads, kv_heads, cos, sin, pos, mask, past_k=None if past is None else past[0]))
        _, past = G.decoder_layer(x.to(dtype), pp, heads, kv_heads, cos, sin, pos, mask, past_kv=past, return_kv=True)
    return outs


def kernel_weights(q, k, causal=True, seqlens=None, kv_mask=None, dtype=torch.float32):
    """The weights `ops.attn_probs` computes, from token-major q [B, Sq, nh, d] and k [B, Skv, nkv, d] (already rotated): causal is
    bottom-right aligned (query i at position Skv - Sq + i), `seqlens` [B] right-pads keys (Sq == Skv), `kv_mask` [B, Skv] 0 = padded
    key; the masks `_prepare_4d_causal_attention_mask` builds for them."""
    B, Sq = q.shape[:2]
    Skv = k.shape[1]
    am = None
    if seqlens is not None:
        am = (torch.arange(Skv)[None] < torch.as_tensor(seqlens)[:, None]).long()
    if kv_mask is not None:
        am = kv_mask.long() if am is None else am * kv_mask.long()
    if causal:
        mask = O.causal_additive_mask_past(B, Sq, Skv - Sq, dtype, am)
    else:
        mask = torch.zeros(B, 1, Sq, Skv, dtype=dtype)
        if am is not None:
            mask = mask.masked_fill((am == 0)[:, None, None, :], torch.finfo(dtype).min)
    return core_weights(q.transpose(1, 2).to(dtype), k.transpose(1, 2).to(dtype), mask)

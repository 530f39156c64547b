"""Attention-probability timings (dev tool, needs one H100): attn_probs_kernel (`output_attentions=True`) next to the attention forward
it follows.  CUDA events around many launches after warm-up; the card's name and power limit are printed with the numbers, because
they are part of them.

    python scripts/attn_probs.py

  * causal, S 2048, 32 q heads, d 128, B in {1, 4}, nkv in {32, 8}: the kernel's time; the bytes it must write (B nh S^2 x 2, the
    whole dense [B, nh, S, S] bf16, zeros above the diagonal included) over that time; the causal QK^T FLOPs (S^2 d per (batch, q
    head)) over that time; and the attention forward's time on the same inputs for scale;
  * one decode step (1 new token against a 2048-row cache), B 8, 32 q heads, d 128, nkv in {32, 8}: kernel time and the K bytes it reads;
  * one Vicuna-7B decoder-layer forward (hidden 4096, inter 11008, 32 heads), B 4, S 2048, with and without output_attentions.
"""
from __future__ import annotations

import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from dreamllm_b200 import ops  # noqa: E402
from scripts.attn_gqa import _card, _time_ms, _views  # noqa: E402

BF = torch.bfloat16
HBM_TBPS = 3.35            # H100 SXM data-sheet HBM3 bandwidth: the bound a store-bound kernel is measured against


def probs(S=2048, nh=32, d=128, iters=20):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 4):
        for nkv in (32, 8):
            buf = torch.randn(B, S, (nh + 2 * nkv) * d, device="cuda", generator=g).to(BF)
            q, k, v = _views(buf, nh, nkv, d)
            _, lse = ops.attn_fwd(q, k, v, causal=True)
            out = torch.empty(B, nh, S, S, device="cuda", dtype=BF)
            t_p = _time_ms(lambda: ops.attn_probs(q, k, lse, causal=True, out=out), iters)
            t_f = _time_ms(lambda: ops.attn_fwd(q, k, v, causal=True), iters)
            nbytes = B * nh * S * S * 2
            flops = 2.0 * S * S * d * B * nh * 0.5
            rows.append(dict(kind="probs", B=B, S=S, nh=nh, nkv=nkv, d=d, probs_ms=round(t_p, 4), written_gb=round(nbytes / 1e9, 3),
                             write_tbps=round(nbytes / t_p / 1e9, 2), hbm_bound_ms=round(nbytes / HBM_TBPS / 1e9, 4),
                             qk_tflops=round(flops / t_p / 1e9, 1), attn_fwd_ms=round(t_f, 4)))
            del buf, out, lse
            torch.cuda.empty_cache()
    return rows


def decode(B=8, L=2048, nh=32, d=128, iters=200):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1)
    for nkv in (32, 8):
        kc = torch.randn(B, L, nkv, d, device="cuda", generator=g).to(BF)
        vc = torch.randn(B, L, nkv, d, device="cuda", generator=g).to(BF)
        q = torch.randn(B, 1, nh, d, device="cuda", generator=g).to(BF)
        _, lse = ops.attn_fwd_cache(q, kc, vc, L, causal=True, return_lse=True)
        out = torch.empty(B, nh, 1, L, device="cuda", dtype=BF)
        t = _time_ms(lambda: ops.attn_probs(q, kc, lse, causal=True, kv_len=L, out=out), iters)
        t_f = _time_ms(lambda: ops.attn_fwd_cache(q, kc, vc, L, causal=True), iters)
        k_bytes = B * L * nkv * d * 2
        rows.append(dict(kind="decode", B=B, cache=L, nh=nh, nkv=nkv, d=d, probs_us=round(t * 1e3, 2), k_bytes=k_bytes,
                         k_gbps=round(k_bytes / t / 1e6, 1), written_bytes=B * nh * L * 2, attn_fwd_us=round(t_f * 1e3, 2)))
        del kc, vc
    return rows


def layer(B=4, S=2048, iters=10):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer
    torch.manual_seed(0)
    cfg = DreamLLMConfig(hidden_size=4096, intermediate_size=11008, num_attention_heads=32, num_hidden_layers=1, max_position_embeddings=4096)
    lay = DreamLLMDecoderLayer(cfg).to(device="cuda", dtype=BF)
    x = (torch.randn(B, S, 4096, device="cuda") * 0.5).to(BF)
    row = dict(kind="layer_fwd", shape="vicuna-7b", B=B, S=S, nh=32)
    with torch.no_grad():
        for oa in (False, True):
            row[f"fwd_ms_output_attentions_{oa}"] = round(_time_ms(lambda: lay(x, output_attentions=oa), iters, warmup=3), 3)
    return [row]


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    card = _card()
    print(f"card: {card}")
    for row in probs() + decode() + layer():
        row["card"] = card
        print(json.dumps(row))


if __name__ == "__main__":
    main()

"""Grouped-query attention timings (dev tool, needs one H100): the attention kernels, one decode step and one decoder layer at
multi-head vs grouped-query head counts.  CUDA events around many launches after warm-up; the card's name and power limit are printed
with the numbers, because they are part of them.

    python scripts/attn_gqa.py

  * attention fwd and bwd, causal, B 4, S 2048, 32 q heads, d 128, nkv in {32, 8, 1}: TFLOP/s counted over the q heads
    (fwd 2 GEMMs, bwd 5, each 2 S^2 d per (batch, q head), halved by the causal mask);
  * one decode step (1 new token against a 2048-row cache), B 8, 32 q heads, d 128, nkv in {32, 8}: the K/V bytes the step has to read
    (B x 2048 x nkv x d x 2 tensors x 2 bytes) and that over the kernel time;
  * one decoder layer fwd + bwd, B 4, S 2048: the Vicuna-7B shape (hidden 4096, inter 11008, 32 / 32 heads) vs the Llama-3-8B shape
    (hidden 4096, inter 14336, 32 / 8 heads, rope_theta 500000).
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from dreamllm_b200 import ops  # noqa: E402

BF = torch.bfloat16


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _time_ms(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _views(buf, nh, nkv, d):
    B, S = buf.shape[:2]
    return (buf[..., :nh * d].view(B, S, nh, d), buf[..., nh * d:(nh + nkv) * d].view(B, S, nkv, d),
            buf[..., (nh + nkv) * d:].view(B, S, nkv, d))


def attention(B=4, S=2048, nh=32, d=128, iters=50):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for nkv in (32, 8, 1):
        buf = torch.randn(B, S, (nh + 2 * nkv) * d, device="cuda", generator=g).to(BF)
        q, k, v = _views(buf, nh, nkv, d)
        out, lse = ops.attn_fwd(q, k, v, causal=True)
        dout = torch.randn(B, S, nh * d, device="cuda", generator=g).to(BF)
        dbuf = torch.empty_like(buf)
        dq, dk, dv = _views(dbuf, nh, nkv, d)
        t_f = _time_ms(lambda: ops.attn_fwd(q, k, v, causal=True), iters)
        t_b = _time_ms(lambda: ops.attn_bwd(dout, q, k, v, out, lse, dq, dk, dv, causal=True), iters)
        gemm = 2.0 * S * S * d * B * nh * 0.5                     # one causal S x S x d GEMM over every (batch, q head)
        rows.append(dict(kind="attn", B=B, S=S, nh=nh, nkv=nkv, d=d, fwd_ms=round(t_f, 4), bwd_ms=round(t_b, 4),
                         fwd_tflops=round(2 * gemm / t_f / 1e9, 1), bwd_tflops=round(5 * gemm / t_b / 1e9, 1)))
        del buf, dbuf, out, lse, dout
    return rows


def decode(B=8, L=2048, nh=32, d=128, iters=200):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1)
    for nkv in (32, 8):
        kc = torch.randn(B, L, nkv, d, device="cuda", generator=g).to(BF)
        vc = torch.randn(B, L, nkv, d, device="cuda", generator=g).to(BF)
        q = torch.randn(B, 1, nh, d, device="cuda", generator=g).to(BF)
        t = _time_ms(lambda: ops.attn_fwd_cache(q, kc, vc, L, causal=True), iters)
        kv_bytes = 2 * B * L * nkv * d * 2
        rows.append(dict(kind="decode", B=B, cache=L, nh=nh, nkv=nkv, d=d, us=round(t * 1e3, 2), kv_bytes=kv_bytes,
                         kv_gbps=round(kv_bytes / t / 1e6, 1)))
        del kc, vc
    return rows


def layer(B=4, S=2048, iters=10):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer
    rows = []
    for name, inter, nkv, theta in (("vicuna-7b", 11008, 32, 10000.0), ("llama-3-8b", 14336, 8, 500000.0)):
        torch.manual_seed(0)
        cfg = DreamLLMConfig(hidden_size=4096, intermediate_size=inter, num_attention_heads=32, num_key_value_heads=nkv,
                             rope_theta=theta, num_hidden_layers=1, max_position_embeddings=4096)
        lay = DreamLLMDecoderLayer(cfg).to(device="cuda", dtype=BF)
        x = (torch.randn(B, S, 4096, device="cuda") * 0.5).to(BF).requires_grad_(True)
        gy = torch.randn(B, S, 4096, device="cuda").to(BF)

        def step():
            for p in lay.parameters():
                p.grad = None
            x.grad = None
            lay(x)[0].backward(gy)
        t = _time_ms(step, iters, warmup=3)
        rows.append(dict(kind="layer", shape=name, B=B, S=S, nh=32, nkv=nkv, inter=inter, fwd_bwd_ms=round(t, 3)))
        del lay, x, gy
        torch.cuda.empty_cache()
    return rows


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    card = _card()
    print(f"card: {card}")
    for row in attention() + decode() + layer():
        row["card"] = card
        print(json.dumps(row))


if __name__ == "__main__":
    main()

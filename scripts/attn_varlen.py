"""Packed against right-padded batches (dev tool, needs one H100): the variable-length attention kernels against the padded ones on
the same ragged lengths, and one decoder layer fwd + bwd in either layout.  CUDA events around many launches after warm-up, the two
sides alternated in rounds; the card's name and power limit are printed with the numbers, because they are part of them.

    python scripts/attn_varlen.py

Length sets (Vicuna-7B heads, 32 x 128, and 32 / 8 grouped-query):
  * uniform    2048 x 4: packing gains nothing here, so this is the overhead of the variable-length path;
  * ragged     2048 / 1200 / 700 / 300: 8192 padded rows for 4248 tokens;
  * skewed     one 2048 and seven short samples: most CTAs of the (max tiles, heads, samples) grid exit at once.
Attention FLOPs are counted over the causal area of the real tokens, sum_b len_b^2 / 2 per GEMM (fwd 2 GEMMs, bwd 5), for both sides:
the padded kernels skip pad keys too, so the two rates are over the same work.  The layer rows report real tokens per second.
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
LENGTHS = {"uniform": [2048] * 4, "ragged": [2048, 1200, 700, 300], "skewed": [2048, 300, 180, 420, 96, 250, 130, 64]}


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _time_pair_ms(fa, fb, iters, rounds=4, warmup=5):
    """ms per call of fa and fb, timed in alternating windows of `iters` launches"""
    for _ in range(warmup):
        fa()
        fb()
    torch.cuda.synchronize()
    tot = [0.0, 0.0]
    for _ in range(rounds):
        for i, fn in enumerate((fa, fb)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            tot[i] += e0.elapsed_time(e1)
    return tot[0] / (rounds * iters), tot[1] / (rounds * iters)


def _heads(buf, nh, nkv):
    return buf[..., :nh, :], buf[..., nh:nh + nkv, :], buf[..., nh + nkv:, :]


def attention(nh=32, d=128, iters=30):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for nkv in (32, 8):
        for name, lens in LENGTHS.items():
            B, S, T = len(lens), max(lens), sum(lens)
            sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
            cu = torch.zeros(B + 1, dtype=torch.int32, device="cuda")
            cu[1:] = sl.cumsum(0)
            pad = torch.randn(B, S, nh + 2 * nkv, d, device="cuda", generator=g).to(BF)
            valid = torch.arange(S, device="cuda")[None] < sl[:, None]
            pk = pad[valid].contiguous()                                           # the same tokens, packed
            dpad = torch.randn(B, S, nh * d, device="cuda", generator=g).to(BF) * valid[..., None]
            dpk = dpad[valid].contiguous()
            qp, kp, vp = _heads(pad, nh, nkv)
            qk, kk, vk = _heads(pk, nh, nkv)
            op, lp = ops.attn_fwd(qp, kp, vp, causal=True, seqlens=sl)
            ok, lk = ops.attn_fwd_varlen(qk, kk, vk, cu, S, causal=True)
            assert torch.equal(op[valid], ok)                                      # same rows, same bits
            gpad, gpk = torch.empty_like(pad), torch.empty_like(pk)
            f_pad, f_pk = _time_pair_ms(lambda: ops.attn_fwd(qp, kp, vp, causal=True, seqlens=sl),
                                        lambda: ops.attn_fwd_varlen(qk, kk, vk, cu, S, causal=True), iters)
            b_pad, b_pk = _time_pair_ms(lambda: ops.attn_bwd(dpad, qp, kp, vp, op, lp, *_heads(gpad, nh, nkv), causal=True, seqlens=sl),
                                        lambda: ops.attn_bwd_varlen(dpk, qk, kk, vk, ok, lk, *_heads(gpk, nh, nkv), cu, S, causal=True),
                                        iters)
            assert torch.equal(gpad[valid], gpk)
            gemm = sum(2.0 * n * n * d * nh * 0.5 for n in lens)                   # one causal GEMM over the real tokens
            rows.append(dict(kind="attn", lengths=name, B=B, S=S, T=T, nh=nh, nkv=nkv, d=d,
                             fwd_ms_padded=round(f_pad, 4), fwd_ms_packed=round(f_pk, 4), bwd_ms_padded=round(b_pad, 4),
                             bwd_ms_packed=round(b_pk, 4), fwd_tflops_padded=round(2 * gemm / f_pad / 1e9, 1),
                             fwd_tflops_packed=round(2 * gemm / f_pk / 1e9, 1), bwd_tflops_padded=round(5 * gemm / b_pad / 1e9, 1),
                             bwd_tflops_packed=round(5 * gemm / b_pk / 1e9, 1)))
            del pad, pk, dpad, dpk, gpad, gpk, op, ok
    return rows


def layer(iters=5):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer
    rows = []
    for shape, inter, nkv in (("vicuna-7b", 11008, 32), ("32/8 gqa", 11008, 8)):
        torch.manual_seed(0)
        cfg = DreamLLMConfig(hidden_size=4096, intermediate_size=inter, num_attention_heads=32, num_key_value_heads=nkv,
                             num_hidden_layers=1, max_position_embeddings=4096)
        lay = DreamLLMDecoderLayer(cfg).to(device="cuda", dtype=BF)
        for name, lens in LENGTHS.items():
            B, S, T = len(lens), max(lens), sum(lens)
            sl = torch.tensor(lens, dtype=torch.int32)
            cu = torch.zeros(B + 1, dtype=torch.int32)
            cu[1:] = sl.cumsum(0)
            cu_dev, sl_dev = cu.cuda(), sl.cuda()
            valid = (torch.arange(S)[None] < sl[:, None]).cuda()
            xp = ((torch.randn(B, S, 4096, device="cuda") * 0.5).to(BF) * valid[..., None]).requires_grad_(True)
            gp = torch.randn(B, S, 4096, device="cuda").to(BF) * valid[..., None]
            xk = xp.detach()[valid][None].contiguous().requires_grad_(True)
            gk = gp[valid][None].contiguous()
            mask = valid.long()

            def clear():
                for p in lay.parameters():
                    p.grad = None
                xp.grad = xk.grad = None

            def padded():
                clear()
                lay(xp, attention_mask=mask, seqlens=sl_dev)[0].backward(gp)

            def packed():
                clear()
                lay(xk, cu_seqlens=cu_dev, max_seqlen=S)[0].backward(gk)
            t_pad, t_pk = _time_pair_ms(padded, packed, iters, rounds=3, warmup=2)
            rows.append(dict(kind="layer", shape=shape, lengths=name, B=B, S=S, T=T, rows_padded=B * S, nkv=nkv,
                             fwd_bwd_ms_padded=round(t_pad, 3), fwd_bwd_ms_packed=round(t_pk, 3),
                             tokens_per_s_padded=round(T / t_pad * 1e3), tokens_per_s_packed=round(T / t_pk * 1e3)))
            del xp, gp, xk, gk
        del lay
        torch.cuda.empty_cache()
    return rows


def main():
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    card = _card()
    print(f"card: {card}")
    for row in attention() + layer():
        row["card"] = card
        print(json.dumps(row))


if __name__ == "__main__":
    main()

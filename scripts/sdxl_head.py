"""SDXL head timings (dev tool, needs one H100): the UNet-XL at 128x128 latents (1024^2 images) with Q = 196 dream queries, randomly
initialised (no checkpoint is read; the timings do not depend on the weights).  CUDA events around warmed-up work; the card's name and
power limit are printed with the numbers, because they are part of them.

    python scripts/sdxl_head.py [--out FILE.json]

  * UNet-XL forward, B 1 / 2 / 4, and its TFLOP/s over the analytic FLOP count of `unet_flops` (GEMMs, convolutions and attention
    products; norms and element-wise work not counted);
  * the training forward with tape + `backward_cond` (conditioning and text_embeds gradients) per sample, B 1 / 2, with the peak memory
    of that step (torch.cuda.max_memory_allocated, UNet weights included);
  * one 50-step CFG sampler loop (DDPM, one captured graph) at B 1 and B 4;
  * VAE encode and decode of one 1024^2 image (bf16).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from dreamllm_b200 import ops  # noqa: E402
from scripts.attn_gqa import _card, _time_ms  # noqa: E402

BF = torch.bfloat16


def unet_flops(unet, B, H, W, Q):
    """Multiply-adds x 2 of one UNet forward: every conv / linear at the resolution it runs at, plus QK^T and PV of self- and
    cross-attention."""
    total = 0.0

    def conv(c, px):
        return 2.0 * px * c.weight.numel()

    def resnet(r, px):
        f = conv(r.conv1, px) + conv(r.conv2, px) + 2.0 * r.time_emb_proj.weight.numel()
        if r.conv_shortcut is not None:
            f += conv(r.conv_shortcut, px)
        return f

    def transformer(t, px):
        C = t.proj_in.weight.shape[0]
        f = 2.0 * px * (t.proj_in.weight.numel() + t.proj_out.weight.numel())
        for blk in t.transformer_blocks:
            lin = (blk.attn1.to_q.weight.numel() * 3 + blk.attn1.to_out[0].weight.numel() + blk.attn2.to_q.weight.numel()
                   + blk.attn2.to_out[0].weight.numel() + blk.ff.net[0].proj.weight.numel() + blk.ff.net[2].weight.numel())
            f += 2.0 * px * lin + 2.0 * B * Q * 2 * blk.attn2.to_k.weight.numel()     # cross K/V (once per prompt)
            f += 4.0 * px * (px // B) * C + 4.0 * px * Q * C                           # self: QK^T + PV per sample; cross
        return f

    px = B * H * W
    total += conv(unet.conv_in, px)
    for b in unet.down_blocks:
        for j, r in enumerate(b.resnets):
            total += resnet(r, px)
            if hasattr(b, "attentions"):
                total += transformer(b.attentions[j], px)
        if hasattr(b, "downsamplers"):
            px //= 4
            total += conv(b.downsamplers[0].conv, px)
    total += resnet(unet.mid_block.resnets[0], px) + transformer(unet.mid_block.attentions[0], px) + resnet(unet.mid_block.resnets[1], px)
    for b in unet.up_blocks:
        for j, r in enumerate(b.resnets):
            total += resnet(r, px)
            if hasattr(b, "attentions"):
                total += transformer(b.attentions[j], px)
        if hasattr(b, "upsamplers"):
            px *= 4
            total += conv(b.upsamplers[0].conv, px)
    total += conv(unet.conv_out, px)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    from dreamllm_b200.unet import SDXL, DenoiseLoop, UNet2DConditionModel
    from dreamllm_b200.vae import AutoencoderKLDecoder, AutoencoderKLEncoder
    torch.manual_seed(0)
    unet = UNet2DConditionModel(SDXL)
    for p in unet.parameters():                      # keep activations in a realistic range with random weights
        if p.dim() > 1:
            p.data.mul_(0.5)
    unet = unet.to(device="cuda", dtype=BF)
    H = W = 128
    Q = 196
    g = torch.Generator(device="cuda").manual_seed(1)
    rec = {"card": _card(), "latents": [H, W], "Q": Q}
    ids = torch.tensor([[1024., 1024., 0., 0., 1024., 1024.]], device="cuda")

    fwd = []
    for B in (1, 2, 4):
        x = torch.randn(B, 4, H, W, device="cuda", generator=g)
        c = (torch.randn(B, Q, 2048, device="cuda", generator=g) * 0.5).to(BF)
        text = torch.randn(B, 1280, device="cuda", generator=g).to(BF)
        add = dict(text_embeds=text, time_ids=ids.repeat(B, 1))
        ms = _time_ms(lambda: unet(x, 500, c, add), 5, warmup=2)
        fl = unet_flops(unet, B, H, W, Q)
        fwd.append({"B": B, "ms": round(ms, 2), "tflop": round(fl / 1e12, 2), "tflops": round(fl / ms / 1e9, 1)})
        print("forward", fwd[-1], flush=True)
    rec["forward"] = fwd

    train = []
    for B in (1, 2):
        x = torch.randn(B, 4, H, W, device="cuda", generator=g)
        c = (torch.randn(B, Q, 2048, device="cuda", generator=g) * 0.5).to(BF)
        text = torch.randn(B, 1280, device="cuda", generator=g).to(BF)
        t = torch.randint(0, 1000, (B,), device="cuda", dtype=torch.int32, generator=g)
        tgt = torch.randn_like(x)

        def step():
            eps, tape = unet.forward_train(x, t, c, (text, ids.repeat(B, 1)))
            _, deps = ops.mse_fwd_bwd(eps, tgt)
            return unet.backward_cond(deps, tape)

        step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ms = _time_ms(step, 3, warmup=1)
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        fl = 3 * unet_flops(unet, B, H, W, Q)          # forward + dgrad (about 2x the forward's products)
        train.append({"B": B, "ms": round(ms, 1), "ms_per_sample": round(ms / B, 1), "peak_gib": round(peak, 2),
                      "tflops_approx": round(fl / ms / 1e9, 1)})
        print("train fwd+backward_cond", train[-1], flush=True)
    rec["train"] = train
    rec["weights_gib"] = round(sum(p.numel() for p in unet.parameters()) * 2 / 2 ** 30, 2)

    loops = []
    for B in (1, 4):
        cond = (torch.randn(2 * B, Q, 2048, device="cuda", generator=g) * 0.5).to(BF)
        text = torch.randn(2 * B, 1280, device="cuda", generator=g).to(BF)
        aug = unet.add_embedding_fwd(text, ids.repeat(2 * B, 1))
        loop = DenoiseLoop(unet, cond, 50, 7.5, "ddpm", height=8 * H, width=8 * W, aug_emb=aug)
        loop.run()                                   # capture + first replay
        torch.cuda.synchronize()
        loop.reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loop.run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        fl = 50 * unet_flops(unet, 2 * B, H, W, Q)
        loops.append({"B": B, "ms": round(ms, 1), "ms_per_step": round(ms / 50, 2), "tflops": round(fl / ms / 1e9, 1)})
        print("50-step CFG loop", loops[-1], flush=True)
        del loop
    rec["loop50_cfg"] = loops
    del unet
    torch.cuda.empty_cache()

    enc = AutoencoderKLEncoder(dict(scaling_factor=0.13025)).to(device="cuda", dtype=BF)
    dec = AutoencoderKLDecoder(dict(scaling_factor=0.13025)).to(device="cuda", dtype=BF)
    img = (torch.rand(1, 3, 1024, 1024, device="cuda", generator=g) * 2 - 1).to(BF)
    lat = torch.randn(1, 4, 128, 128, device="cuda", generator=g) * 0.13025
    rec["vae_encode_ms"] = round(_time_ms(lambda: enc.encode_sample(img), 5, warmup=2), 2)
    rec["vae_decode_ms"] = round(_time_ms(lambda: dec.decode(lat), 5, warmup=2), 2)
    print("vae", rec["vae_encode_ms"], rec["vae_decode_ms"], flush=True)
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE ONLY — from-spec CPU restatement of the SDXL-base `UNet2DConditionModel` (diffusers 0.24).

Extends oracle/unet_oracle.py (SD-2.1) with what SDXL adds, restated from diffusers' unet_2d_condition.py / transformer_2d.py /
embeddings.py and the SDXL-base unet/config.json:
  * `transformer_layers_per_block` (per level; the mid block takes the last, the up blocks the reversed list): a Transformer2DModel holds
    that many BasicTransformerBlocks, applied in sequence between proj_in and proj_out;
  * `addition_embed_type "text_time"`: aug = add_embedding(cat(text_embeds, Timesteps(256)(time_ids.flatten()).reshape(B, -1)).to(dtype)),
    emb = time_embedding(t) + aug.
With the default config it builds exactly the SD-2.1 UNet of unet_oracle.py (same keys, same arithmetic).  Validated by the parameter
count (2 567 463 684 = the published SDXL-base UNet size) and key agreement with the native module.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import unet_oracle as UO

SDXL = dict(in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280), layers_per_block=2, attention_head_dim=(5, 10, 20),
            cross_attention_dim=2048, norm_num_groups=32, norm_eps=1e-5, down_attn=(False, True, True), up_attn=(True, True, False),
            transformer_layers_per_block=(1, 2, 10), addition_embed_type="text_time", addition_time_embed_dim=256,
            projection_class_embeddings_input_dim=2816)


class Transformer2DModel(UO.Transformer2DModel):
    def __init__(self, dim, heads, ctx_dim, groups=32, depth=1):
        super().__init__(dim, heads, ctx_dim, groups)
        self.transformer_blocks = nn.ModuleList([UO.BasicTransformerBlock(dim, heads, ctx_dim) for _ in range(depth)])

    def forward(self, x, ctx):
        B, C, H, W = x.shape
        h = self.proj_in(self.norm(x).permute(0, 2, 3, 1).reshape(B, H * W, C))
        for blk in self.transformer_blocks:
            h = blk(h, ctx)
        return self.proj_out(h).reshape(B, H, W, C).permute(0, 3, 1, 2) + x


class UNet2DConditionModel(nn.Module):
    def __init__(self, cfg=None):
        super().__init__()
        c = dict(UO.SD21)
        c.update(cfg or {})
        self.cfg = c
        ch, heads, ctx, G, L = c["block_out_channels"], c["attention_head_dim"], c["cross_attention_dim"], c["norm_num_groups"], c["layers_per_block"]
        depth = tuple(c.get("transformer_layers_per_block") or (1,) * len(ch))
        temb = ch[0] * 4
        self.conv_in = nn.Conv2d(c["in_channels"], ch[0], 3, padding=1)
        self.time_embedding = UO.TimestepEmbedding(ch[0], temb)
        if c.get("addition_embed_type") == "text_time":
            self.add_embedding = UO.TimestepEmbedding(c["projection_class_embeddings_input_dim"], temb)
        else:
            self.add_embedding = None
        self.down_blocks = nn.ModuleList()
        out = ch[0]
        for i, co in enumerate(ch):
            b = UO._Block()
            cin, out = out, co
            b.resnets = nn.ModuleList([UO.ResnetBlock2D(cin if j == 0 else out, out, temb, G) for j in range(L)])
            if c["down_attn"][i]:
                b.attentions = nn.ModuleList([Transformer2DModel(out, heads[i], ctx, G, depth[i]) for _ in range(L)])
            if i < len(ch) - 1:
                b.downsamplers = nn.ModuleList([UO.Downsample2D(out)])
            self.down_blocks.append(b)
        self.mid_block = UO._Block()
        self.mid_block.resnets = nn.ModuleList([UO.ResnetBlock2D(ch[-1], ch[-1], temb, G), UO.ResnetBlock2D(ch[-1], ch[-1], temb, G)])
        self.mid_block.attentions = nn.ModuleList([Transformer2DModel(ch[-1], heads[-1], ctx, G, depth[-1])])
        self.up_blocks = nn.ModuleList()
        rev, rheads, rdepth = list(reversed(ch)), list(reversed(heads)), list(reversed(depth))
        prev = rev[0]
        for i, co in enumerate(rev):
            b = UO._Block()
            skip_in = rev[min(i + 1, len(ch) - 1)]
            b.resnets = nn.ModuleList([UO.ResnetBlock2D((prev if j == 0 else co) + (skip_in if j == L else co), co, temb, G)
                                       for j in range(L + 1)])
            if c["up_attn"][i]:
                b.attentions = nn.ModuleList([Transformer2DModel(co, rheads[i], ctx, G, rdepth[i]) for _ in range(L + 1)])
            if i < len(ch) - 1:
                b.upsamplers = nn.ModuleList([UO.Upsample2D(co)])
            prev = co
            self.up_blocks.append(b)
        self.conv_norm_out = nn.GroupNorm(G, ch[0], eps=c["norm_eps"])
        self.conv_out = nn.Conv2d(ch[0], c["out_channels"], 3, padding=1)

    def add_embeds(self, text_embeds, time_ids, dtype):
        """cat(text_embeds, Timesteps(addition_time_embed_dim)(time_ids)) rounded once to `dtype` (the sinusoid is fp32)."""
        B = text_embeds.shape[0]
        te = UO.timestep_embedding(time_ids.flatten(), self.cfg["addition_time_embed_dim"]).reshape(B, -1)
        return torch.cat([text_embeds.float(), te], dim=-1).to(dtype)

    def forward(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=None):
        B = sample.shape[0]
        t = torch.as_tensor(timestep)
        t = t.expand(B) if t.dim() == 0 else t
        temb = self.time_embedding(UO.timestep_embedding(t, self.cfg["block_out_channels"][0]).to(sample.dtype))
        if self.add_embedding is not None:
            add = self.add_embeds(added_cond_kwargs["text_embeds"], added_cond_kwargs["time_ids"], temb.dtype)
            temb = temb + self.add_embedding(add)
        x = self.conv_in(sample)
        skips = [x]
        for b in self.down_blocks:
            for j, r in enumerate(b.resnets):
                x = r(x, temb)
                if hasattr(b, "attentions"):
                    x = b.attentions[j](x, encoder_hidden_states)
                skips.append(x)
            if hasattr(b, "downsamplers"):
                x = b.downsamplers[0](x)
                skips.append(x)
        x = self.mid_block.resnets[0](x, temb)
        x = self.mid_block.attentions[0](x, encoder_hidden_states)
        x = self.mid_block.resnets[1](x, temb)
        for b in self.up_blocks:
            for j, r in enumerate(b.resnets):
                x = r(torch.cat([x, skips.pop()], dim=1), temb)
                if hasattr(b, "attentions"):
                    x = b.attentions[j](x, encoder_hidden_states)
            if hasattr(b, "upsamplers"):
                x = b.upsamplers[0](x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))

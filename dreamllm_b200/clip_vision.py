"""H100-native CLIP ViT vision tower (forward only), state-dict compatible with `transformers.CLIPVisionModel`.

Reference call site: `CLIPVisionEmbedding.forward`, modeling_plugins.py:321-323 —
    output = self.clip_vision_model(images, output_hidden_states=True); hidden_states[select_layer][:, 1:]
The arithmetic lives in transformers==4.35.2 `modeling_clip.py` (CLIPVisionEmbeddings / CLIPEncoderLayer / CLIPAttention /
CLIPMLP), restated per SURVEY.md Appendix A.4: conv patch-embed (k=s=patch, no bias) + CLS + learned pos-emb ->
pre_layrnorm -> L x { x += out_proj(attn(LN1 x)) ; x += fc2(quick_gelu(fc1(LN2 x))) }.

Kernels: patch-embed = unfold + wgmma GEMM; fused q|k|v GEMM (+bias); non-causal wgmma flash attention d=64;
out_proj / fc2 GEMMs with bias+residual epilogue; fc1 GEMM with bias+quick_gelu epilogue; LayerNorm kernel.
Layers after `select_layer` are never computed (the reference runs and discards them, SURVEY §8 row a11).
The tower is frozen on this path (freeze_clip_vision_model=True, configs/common.py:35) -> runs under no_grad.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops
from .modeling_dreamllm import _fuse_rows

BF16 = torch.bfloat16


class CLIPVisionConfigLite(SimpleNamespace):
    """Fields of transformers.CLIPVisionConfig that the tower reads (ViT-L/14: 1024/24/16/4096, patch 14)."""

    def __init__(self, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16, image_size=224,
                 patch_size=14, layer_norm_eps=1e-5, hidden_act="quick_gelu", num_channels=3, **kw):
        super().__init__(hidden_size=hidden_size, intermediate_size=intermediate_size, num_hidden_layers=num_hidden_layers,
                         num_attention_heads=num_attention_heads, image_size=image_size, patch_size=patch_size,
                         layer_norm_eps=layer_norm_eps, hidden_act=hidden_act, num_channels=num_channels, **kw)

    def to_dict(self):
        return dict(self.__dict__)


class _Embeddings(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.class_embedding = nn.Parameter(torch.randn(c.hidden_size))
        self.patch_embedding = nn.Conv2d(c.num_channels, c.hidden_size, kernel_size=c.patch_size, stride=c.patch_size, bias=False)
        self.num_patches = (c.image_size // c.patch_size) ** 2
        self.num_positions = self.num_patches + 1
        self.position_embedding = nn.Embedding(self.num_positions, c.hidden_size)
        self.register_buffer("position_ids", torch.arange(self.num_positions).expand((1, -1)), persistent=False)


class _Attention(nn.Module):
    def __init__(self, c):
        super().__init__()
        H = c.hidden_size
        self.k_proj = nn.Linear(H, H)
        self.v_proj = nn.Linear(H, H)
        self.q_proj = nn.Linear(H, H)
        self.out_proj = nn.Linear(H, H)


class _MLP(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.fc1 = nn.Linear(c.hidden_size, c.intermediate_size)
        self.fc2 = nn.Linear(c.intermediate_size, c.hidden_size)


class _EncoderLayer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.self_attn = _Attention(c)
        self.layer_norm1 = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
        self.mlp = _MLP(c)
        self.layer_norm2 = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)


class _Encoder(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.layers = nn.ModuleList([_EncoderLayer(c) for _ in range(c.num_hidden_layers)])


class _VisionTransformer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.embeddings = _Embeddings(c)
        self.pre_layrnorm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)  # (sic) — transformers' spelling
        self.encoder = _Encoder(c)
        self.post_layernorm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)


class CLIPVisionModel(nn.Module):
    """Drop-in for `transformers.CLIPVisionModel` as used by CLIPVisionEmbedding (same parameter names)."""

    def __init__(self, config):
        super().__init__()
        if getattr(config, "hidden_act", "quick_gelu") != "quick_gelu":
            raise ValueError("only quick_gelu CLIP towers are supported (ViT-L/14 family)")
        if (config.hidden_size // config.num_attention_heads) != 64:
            raise ValueError("CLIP head_dim must be 64")
        self.config = config
        self.vision_model = _VisionTransformer(config)
        self._wpatch = None

    @property
    def device(self):
        return self.vision_model.pre_layrnorm.weight.device

    @property
    def dtype(self):
        return self.vision_model.pre_layrnorm.weight.dtype

    def _patch_weight(self):
        """conv weight [C,3,p,p] -> [C, Kpad] (flatten order (c,ky,kx), zero-padded to a multiple of 8)."""
        w = self.vision_model.embeddings.patch_embedding.weight
        K = w[0].numel()
        kpad = (K + 7) // 8 * 8
        ver = (w.data_ptr(), w._version)
        if self._wpatch is None or self._wpatch[0] != ver:
            wp = torch.zeros((w.shape[0], kpad), device=w.device, dtype=BF16)
            wp[:, :K] = w.detach().reshape(w.shape[0], K)
            self._wpatch = (ver, wp, kpad)
        return self._wpatch[1], self._wpatch[2]

    @torch.no_grad()
    def hidden_state(self, pixel_values: torch.Tensor, select_layer: int = -2) -> torch.Tensor:
        """== transformers' `model(pixel_values, output_hidden_states=True).hidden_states[select_layer]`."""
        c = self.config
        vm = self.vision_model
        if not pixel_values.is_cuda:
            raise RuntimeError("dreamllm_b200 CLIP tower requires CUDA tensors; there is no CPU fallback")
        x = pixel_values.to(BF16).contiguous()
        N = x.shape[0]
        if x.shape[-1] != c.image_size or x.shape[-2] != c.image_size:
            raise ValueError(f"Input image size ({x.shape[-2]}*{x.shape[-1]}) doesn't match model ({c.image_size}*{c.image_size}).")
        wp, kpad = self._patch_weight()
        P = vm.embeddings.num_patches
        patches = ops.clip_patchify(x, c.patch_size, kpad)                          # [N*P, kpad]
        pe = ops.linear(patches, wp)                                                # [N*P, C]
        h = ops.clip_assemble(pe, vm.embeddings.class_embedding, vm.embeddings.position_embedding.weight, N, P)
        S, C, nh = P + 1, c.hidden_size, c.num_attention_heads
        T = N * S
        h = ops.layernorm_fwd(h.view(T, C), vm.pre_layrnorm.weight, vm.pre_layrnorm.bias, c.layer_norm_eps)
        n_layers = c.num_hidden_layers
        idx = select_layer if select_layer >= 0 else n_layers + 1 + select_layer     # hidden_states has n_layers + 1 entries
        if not 0 <= idx <= n_layers:
            raise IndexError("select_layer out of range")
        for li in range(idx):                                                       # layers >= idx never influence the result
            lyr = vm.encoder.layers[li]
            a = lyr.self_attn
            wqkv = _fuse_rows([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight])
            bqkv = _fuse_rows([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias])
            y = ops.layernorm_fwd(h, lyr.layer_norm1.weight, lyr.layer_norm1.bias, c.layer_norm_eps)
            qkv = ops.linear(y, wqkv, bias=bqkv).view(N, S, 3, nh, 64)
            ao, _ = ops.attn_fwd(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], causal=False)
            h = ops.linear(ao.view(T, C), a.out_proj.weight, bias=a.out_proj.bias, residual=h)
            y = ops.layernorm_fwd(h, lyr.layer_norm2.weight, lyr.layer_norm2.bias, c.layer_norm_eps)
            f = ops.linear(y, lyr.mlp.fc1.weight, bias=lyr.mlp.fc1.bias, act=ops.ACT_QUICK_GELU)
            h = ops.linear(f, lyr.mlp.fc2.weight, bias=lyr.mlp.fc2.bias, residual=h)
        return h.view(N, S, C)

    def forward(self, pixel_values, output_hidden_states=True, select_layer=-2, **kw):
        hs = self.hidden_state(pixel_values, select_layer)
        return SimpleNamespace(last_hidden_state=None, pooler_output=None, hidden_states={select_layer: hs})

"""H100-native CLIP ViT vision tower, state-dict compatible with `transformers.CLIPVisionModel`.

Reference call site: `CLIPVisionEmbedding.forward`, modeling_plugins.py:321-323 —
    output = self.clip_vision_model(images, output_hidden_states=True); hidden_states[select_layer][:, 1:]
The arithmetic lives in transformers==4.35.2 `modeling_clip.py` (CLIPVisionEmbeddings / CLIPEncoderLayer / CLIPAttention /
CLIPMLP), restated per SURVEY.md Appendix A.4: conv patch-embed (k=s=patch, no bias) + CLS + learned pos-emb ->
pre_layrnorm -> L x { x += out_proj(attn(LN1 x)) ; x += fc2(quick_gelu(fc1(LN2 x))) }.

Kernels: patch-embed = unfold + wgmma GEMM; fused q|k|v GEMM (+bias); non-causal wgmma flash attention d=64;
out_proj / fc2 GEMMs with bias+residual epilogue; fc1 GEMM with bias+quick_gelu epilogue; LayerNorm kernel.
Layers after `select_layer` are never computed (the reference runs and discards them, SURVEY §8 row a11).

Two paths, chosen by whether any tower parameter requires grad:
* frozen (every shipped config, freeze_clip_vision_model=True, configs/common.py:35): runs under no_grad with the fused quick-GELU
  epilogue and the row-fused q|k|v weight (`_fuse_rows`);
* trainable (freeze_clip_vision_model=False and/or freeze_embedding_layers=False): per-layer autograd Functions.  fc1 runs as a
  bias-only GEMM whose bf16 output is kept for the backward and a separate quick-GELU kernel applies the activation (where
  transformers rounds), so its features may differ from the frozen path's in the last bit.  Parameters are never re-seated (a
  gradient reducer / sharded optimizer owns their storage): q|k|v are gathered into a per-forward buffer instead.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
import torch.nn as nn

from . import ops
from .ddp import grad_out_view
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
        """conv weight [C,3,p,p] -> [C, Kpad] (flatten order (c,ky,kx), zero-padded to a multiple of 8).  A trainable or optimizer-owned
        weight is rebuilt on every call: the AdamW kernel writes parameters through raw pointers without bumping `_version`, so the
        cache key would not see the update."""
        w = self.vision_model.embeddings.patch_embedding.weight
        K = w[0].numel()
        kpad = (K + 7) // 8 * 8
        ver = (w.data_ptr(), w._version)
        if self._wpatch is None or self._wpatch[0] != ver or w.requires_grad or hasattr(w, "_dllm_grad_view"):
            wp = torch.zeros((w.shape[0], kpad), device=w.device, dtype=BF16)
            wp[:, :K] = w.detach().reshape(w.shape[0], K)
            self._wpatch = (ver, wp, kpad)
        return self._wpatch[1], self._wpatch[2]

    def _check_input(self, pixel_values, select_layer):
        c = self.config
        if not pixel_values.is_cuda:
            raise RuntimeError("dreamllm_b200 CLIP tower requires CUDA tensors; there is no CPU fallback")
        x = pixel_values.to(BF16).contiguous()
        if x.shape[-1] != c.image_size or x.shape[-2] != c.image_size:
            raise ValueError(f"Input image size ({x.shape[-2]}*{x.shape[-1]}) doesn't match model ({c.image_size}*{c.image_size}).")
        n_layers = c.num_hidden_layers
        idx = select_layer if select_layer >= 0 else n_layers + 1 + select_layer     # hidden_states has n_layers + 1 entries
        if not 0 <= idx <= n_layers:
            raise IndexError("select_layer out of range")
        return x, idx

    def hidden_state(self, pixel_values: torch.Tensor, select_layer: int = -2) -> torch.Tensor:
        """== transformers' `model(pixel_values, output_hidden_states=True).hidden_states[select_layer]`.  Differentiable with respect to
        the tower parameters that require grad (none: the no_grad path below, with the fused epilogues)."""
        # The choice ignores grad mode on purpose: under no_grad (evaluation, generate) a trainable tower still runs the training
        # forward, so its features carry the same bits as in training and its parameters are never re-seated.
        if any(p.requires_grad for p in self.parameters()):
            return self._hidden_state_train(pixel_values, select_layer)
        return self._hidden_state_frozen(pixel_values, select_layer)

    @torch.no_grad()
    def _hidden_state_frozen(self, pixel_values, select_layer):
        c = self.config
        vm = self.vision_model
        x, idx = self._check_input(pixel_values, select_layer)
        N = x.shape[0]
        # parameters a gradient reducer / sharded optimizer owns (a trainable tower whose flags are off for this call) stay in their
        # buckets: q|k|v are gathered instead of re-seated, and deferred all-gathers are waited for before the weights are read
        owned = any(hasattr(p, "_dllm_grad_view") for p in self.parameters())
        if owned:
            _run_pre_hooks(vm.embeddings, vm.pre_layrnorm)
        wp, kpad = self._patch_weight()
        P = vm.embeddings.num_patches
        patches = ops.clip_patchify(x, c.patch_size, kpad)                          # [N*P, kpad]
        pe = ops.linear(patches, wp)                                                # [N*P, C]
        h = ops.clip_assemble(pe, vm.embeddings.class_embedding, vm.embeddings.position_embedding.weight, N, P)
        S, C, nh = P + 1, c.hidden_size, c.num_attention_heads
        T = N * S
        h = ops.layernorm_fwd(h.view(T, C), vm.pre_layrnorm.weight, vm.pre_layrnorm.bias, c.layer_norm_eps)
        for li in range(idx):                                                       # layers >= idx never influence the result
            lyr = vm.encoder.layers[li]
            a = lyr.self_attn
            if owned:
                _run_pre_hooks(lyr)
            gather = torch.cat if owned else _fuse_rows
            wqkv = gather([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight])
            bqkv = gather([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias])
            y = ops.layernorm_fwd(h, lyr.layer_norm1.weight, lyr.layer_norm1.bias, c.layer_norm_eps)
            qkv = ops.linear(y, wqkv, bias=bqkv).view(N, S, 3, nh, 64)
            ao, _ = ops.attn_fwd(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], causal=False)
            h = ops.linear(ao.view(T, C), a.out_proj.weight, bias=a.out_proj.bias, residual=h)
            y = ops.layernorm_fwd(h, lyr.layer_norm2.weight, lyr.layer_norm2.bias, c.layer_norm_eps)
            f = ops.linear(y, lyr.mlp.fc1.weight, bias=lyr.mlp.fc1.bias, act=ops.ACT_QUICK_GELU)
            h = ops.linear(f, lyr.mlp.fc2.weight, bias=lyr.mlp.fc2.bias, residual=h)
        return h.view(N, S, C)

    def _hidden_state_train(self, pixel_values, select_layer):
        c = self.config
        vm = self.vision_model
        x, idx = self._check_input(pixel_values, select_layer)
        emb = vm.embeddings
        _run_pre_hooks(emb, vm.pre_layrnorm)
        wp, kpad = self._patch_weight()
        N, P, C = x.shape[0], emb.num_patches, c.hidden_size
        S = P + 1
        T = N * S
        meta = SimpleNamespace(N=N, P=P, patch=c.patch_size, kpad=kpad, wp=wp, params=(emb.patch_embedding.weight,
                               emb.class_embedding, emb.position_embedding.weight))
        h = _CLIPEmbedFn.apply(x, *meta.params, meta)
        h = _LayerNormFn.apply(h.view(T, C), vm.pre_layrnorm.weight, vm.pre_layrnorm.bias, c.layer_norm_eps)
        for li in range(idx):                                                       # layers >= idx never influence the result
            lyr = vm.encoder.layers[li]
            _run_pre_hooks(lyr)
            params = _layer_params(lyr)
            meta = SimpleNamespace(N=N, S=S, nh=c.num_attention_heads, eps=c.layer_norm_eps, params=params)
            h = _CLIPLayerFn.apply(h, *params, meta)
        return h.view(N, S, C)

    def forward(self, pixel_values, output_hidden_states=True, select_layer=-2, **kw):
        hs = self.hidden_state(pixel_values, select_layer)
        return SimpleNamespace(last_hidden_state=None, pooler_output=None, hidden_states={select_layer: hs})


# ------------------------------------------------------------------------------------------------ trainable tower
def _run_pre_hooks(*modules):
    """The tower reads these modules' parameters without calling the modules, so it runs their forward pre-hooks itself: that is where
    `zero.ShardedAdamW.attach` waits for a bucket's deferred all-gather (`step(defer_gather=True)`).  Each module-level pre-hook is
    called as for a call without arguments, `hook(module, ())`, or `hook(module, (), {})` if it was registered with `with_kwargs=True`;
    return values are ignored (there are no arguments to replace).  Global pre-hooks (`register_module_forward_pre_hook`) are not run."""
    for mod in modules:
        for m in mod.modules():
            for hid, hook in tuple(m._forward_pre_hooks.items()):
                if hid in m._forward_pre_hooks_with_kwargs:
                    hook(m, (), {})
                else:
                    hook(m, ())


def _layer_params(lyr):
    a = lyr.self_attn
    return (lyr.layer_norm1.weight, lyr.layer_norm1.bias, a.q_proj.weight, a.q_proj.bias, a.k_proj.weight, a.k_proj.bias,
            a.v_proj.weight, a.v_proj.bias, a.out_proj.weight, a.out_proj.bias, lyr.layer_norm2.weight, lyr.layer_norm2.bias,
            lyr.mlp.fc1.weight, lyr.mlp.fc1.bias, lyr.mlp.fc2.weight, lyr.mlp.fc2.bias)


def _bias_grad(dy2d, p):
    """Column sum of a GEMM's output gradient [T, n] as bf16 (deterministic), into p's gradient-bucket slice when it has one."""
    out = grad_out_view((p,))
    n = dy2d.shape[1]
    return ops.channel_sum_nhwc(dy2d.view(1, -1, n), out=None if out is None else out.view(1, n), out_dtype=BF16).view(n)


def _ln_bwd(dy, x, w, b, eps, dres, need_w, need_b):
    """dx (+ dres) of a LayerNorm, with the weight / bias gradients when either is trainable (same dx bits either way)."""
    if not (need_w or need_b):
        return ops.layernorm_bwd(dy, x, w, eps, dres=dres), None, None
    dx, dw, db = ops.layernorm_bwd_affine(dy, x, w, eps, dres=dres, dgamma=grad_out_view((w,)), dbeta=grad_out_view((b,)))
    return dx, (dw if need_w else None), (db if need_b else None)


class _CLIPEmbedFn(torch.autograd.Function):
    """Patch conv (unfold + GEMM) + class token + position embedding -> [N, S, C].  Backward: position_embedding's gradient is the
    column sum of dh viewed as [N, S*C], class_embedding's is its row 0, and the patch weight's is wgrad(dh[:, 1:], patches)."""

    @staticmethod
    def forward(ctx, x, w_patch, cls, pos, meta):
        patches = ops.clip_patchify(x, meta.patch, meta.kpad)                                  # [N*P, kpad]
        pe = ops.linear(patches, meta.wp)
        h = ops.clip_assemble(pe, cls, pos, meta.N, meta.P)
        ctx.save_for_backward(patches if ctx.needs_input_grad[1] else None)
        ctx.meta = meta
        return h

    @staticmethod
    def backward(ctx, dh):
        (patches,) = ctx.saved_tensors
        meta = ctx.meta
        w_patch, cls, pos = meta.params
        need = ctx.needs_input_grad
        N, S, C = dh.shape
        dh = dh.contiguous()
        dw = dcls = dpos = None
        if need[2] or need[3]:
            out = grad_out_view((pos,)) if need[3] else None
            dsum = ops.channel_sum_nhwc(dh.view(1, N, S * C), out=None if out is None else out.view(1, S * C), out_dtype=BF16).view(S, C)
            dpos = dsum if need[3] else None
            dcls = dsum[0].clone() if need[2] else None
        if need[1]:
            dpe = dh[:, 1:].reshape(N * meta.P, C)
            dwp = ops.linear_wgrad(dpe, patches)                                                # [C, kpad]
            dw = dwp[:, :w_patch[0].numel()].reshape(w_patch.shape)
        return None, dw, dcls, dpos, None


class _LayerNormFn(torch.autograd.Function):
    """pre_layrnorm on [T, C]."""

    @staticmethod
    def forward(ctx, x, w, b, eps):
        ctx.save_for_backward(x, w, b)
        ctx.eps = eps
        return ops.layernorm_fwd(x, w, b, eps)

    @staticmethod
    def backward(ctx, dy):
        x, w, b = ctx.saved_tensors
        need = ctx.needs_input_grad
        dx, dw, db = _ln_bwd(dy.contiguous(), x, w, b, ctx.eps, None, need[1], need[2])
        return (dx if need[0] else None), dw, db, None


class _CLIPLayerFn(torch.autograd.Function):
    """One CLIPEncoderLayer on h [T, C] (T = N * S tokens).

    fwd: LN1 -> q|k|v GEMM (+bias, weight gathered per forward) -> flash attention (non-causal, d 64) -> out_proj (+bias, +h)
         -> LN2 -> fc1 (+bias) -> quick_gelu -> fc2 (+bias, +h1)
    tape: h, qkv, attention out and lse, h1, the fc1 pre-activation (bf16) and the gathered q|k|v weight; the LayerNorm outputs and the
    activation are recomputed in backward.  Per token that is 10 C bf16 values (C = hidden size, I = 4 C) plus nh fp32.
    bwd: the transposed sequence.  A parameter's gradient is computed only if it requires grad; weight gradients are written straight
    into their gradient-bucket slices (`ddp.grad_out_view`), q / k / v as three column slices of d(qkv); a bias gradient is the column
    sum of its GEMM's output gradient, except k_proj.bias, whose gradient is exactly zero.  The dgrad below the attention block runs only when something below needs it.
    """

    @staticmethod
    def forward(ctx, h, ln1w, ln1b, wq, bq, wk, bk, wv, bv, wo, bo, ln2w, ln2b, w1, b1, w2, b2, meta):
        N, S, nh = meta.N, meta.S, meta.nh
        T, C = h.shape
        wqkv = torch.cat([wq, wk, wv])                      # the parameters keep their own storage (bucket views)
        bqkv = torch.cat([bq, bk, bv])
        y1 = ops.layernorm_fwd(h, ln1w, ln1b, meta.eps)
        qkv = ops.linear(y1, wqkv, bias=bqkv)
        del y1
        q5 = qkv.view(N, S, 3, nh, 64)
        ao, lse = ops.attn_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], causal=False)
        ao = ao.view(T, C)
        h1 = ops.linear(ao, wo, bias=bo, residual=h)
        y2 = ops.layernorm_fwd(h1, ln2w, ln2b, meta.eps)
        f = ops.linear(y2, w1, bias=b1)                     # pre-activation, kept for the backward
        del y2
        act = ops.quick_gelu(f)
        h2 = ops.linear(act, w2, bias=b2, residual=h1)
        ctx.save_for_backward(h, qkv, ao, lse, h1, f, wqkv)
        ctx.meta = meta
        return h2

    @staticmethod
    def backward(ctx, dh2):
        h, qkv, ao, lse, h1, f, wqkv = ctx.saved_tensors
        meta = ctx.meta
        ln1w, ln1b, wq, bq, wk, bk, wv, bv, wo, bo, ln2w, ln2b, w1, b1, w2, b2 = meta.params
        N, S, nh, eps = meta.N, meta.S, meta.nh, meta.eps
        T, C = h.shape
        need = ctx.needs_input_grad
        need_attn = need[0] or any(need[1:11])              # anything at or below the attention block
        dh2 = dh2.contiguous()
        g = [None] * 16
        # ---- MLP
        if need[15]:
            g[14] = ops.linear_wgrad(dh2, ops.quick_gelu(f), out=grad_out_view((w2,)))
        if need[16]:
            g[15] = _bias_grad(dh2, b2)
        if not (need_attn or any(need[11:15])):
            return (None, *g, None)
        df = ops.quick_gelu_bwd(ops.linear_dgrad(dh2, w2), f)
        if need[13]:
            g[12] = ops.linear_wgrad(df, ops.layernorm_fwd(h1, ln2w, ln2b, eps), out=grad_out_view((w1,)))
        if need[14]:
            g[13] = _bias_grad(df, b1)
        if not (need_attn or need[11] or need[12]):
            return (None, *g, None)
        dh1, g[10], g[11] = _ln_bwd(ops.linear_dgrad(df, w1), h1, ln2w, ln2b, eps, dh2, need[11], need[12])
        del df
        if not need_attn:
            return (None, *g, None)
        # ---- attention
        if need[9]:
            g[8] = ops.linear_wgrad(dh1, ao, out=grad_out_view((wo,)))
        if need[10]:
            g[9] = _bias_grad(dh1, bo)
        dao = ops.linear_dgrad(dh1, wo)
        dqkv = torch.empty_like(qkv)
        q5, d5 = qkv.view(N, S, 3, nh, 64), dqkv.view(N, S, 3, nh, 64)
        ops.attn_bwd(dao.view(N, S, C), q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], ao.view(N, S, C), lse, d5[:, :, 0], d5[:, :, 1],
                     d5[:, :, 2], causal=False)
        del dao
        if need[3] or need[5] or need[7]:
            y1 = ops.layernorm_fwd(h, ln1w, ln1b, eps)
            for i, (w, k) in enumerate(((wq, 3), (wk, 5), (wv, 7))):
                if need[k]:
                    g[k - 1] = ops.linear_wgrad(dqkv[:, i * C:(i + 1) * C], y1, out=grad_out_view((w,)))
            del y1
        if need[4] or need[8]:
            dbqkv = ops.channel_sum_nhwc(dqkv.view(1, T, 3 * C), out_dtype=BF16).view(3 * C)
            for i, k in ((0, 4), (2, 8)):
                if need[k]:
                    g[k - 1] = dbqkv[i * C:(i + 1) * C].clone()
        if need[6]:
            # k_proj.bias adds the same q.b_k to every logit of a softmax row, so its gradient is exactly zero.  The column sum of dK
            # would hold only rounding noise: the attention backward forms rowsum(dO * O) from the bf16 O, so the rows of dS do not
            # sum to zero exactly (at ViT-L/14-336 that noise is 6x what transformers' bf16 autograd leaves).
            out = grad_out_view((bk,))
            g[5] = torch.zeros_like(bk) if out is None else out.zero_()
        dh = None
        if need[0] or need[1] or need[2]:
            dh, g[0], g[1] = _ln_bwd(ops.linear_dgrad(dqkv, wqkv), h, ln1w, ln1b, eps, dh1, need[1], need[2])
        return (dh if need[0] else None, *g, None)

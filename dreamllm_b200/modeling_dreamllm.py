"""H100-native mirror of the reference's `omni/models/dreamllm/modeling_dreamllm.py` decoder stack.

Same class names, constructor / forward signatures, parameter names and state-dict keys as the reference
(SURVEY.md §8b) so the classes drop into `omni.models.dreamllm`; all arithmetic runs in libdreamllm_sm100.so.

    DreamLLMRMSNorm            reference modeling_dreamllm.py:77-91
    RotaryEmbedding            :97-128
    DreamLLMMLP                :212-239
    DreamLLMAttention          :254-400  (DreamLLMFlashAttention2 :403-583 is the same math)
    DreamLLMDecoderLayer       :586-654
    DreamLLMModel              :803-1043  (text / inputs_embeds path; plugin splice lives in modeling_plugins)
    DreamLLMForCausalMLM       :1209-1509 (lm_head + shifted masked CE)

There is no eager/CPU fallback: modules raise if their tensors are not on a CUDA device.
"""
from __future__ import annotations

import functools
import logging
import math
from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.utils.checkpoint

from . import ops
from .ddp import grad_out_view

BF16 = torch.bfloat16
logger = logging.getLogger(__name__)


@functools.lru_cache(maxsize=None)
def _warn_once(msg: str):
    """transformers' `logger.warning_once`."""
    logger.warning(msg)


# ------------------------------------------------------------------------------------------------ config
from .configuration_dreamllm import DreamLLMConfig, deep_instantiate  # noqa: E402  (re-exported: the reference keeps it next door too)


def _check_supported(config):
    if getattr(config, "pretraining_tp", 1) != 1:
        raise ValueError("pretraining_tp > 1 is out of scope (SURVEY.md §8a row a6)")
    nkv = getattr(config, "num_key_value_heads", config.num_attention_heads)
    if nkv <= 0 or config.num_attention_heads % nkv != 0:
        raise ValueError(f"num_attention_heads ({config.num_attention_heads}) must be a multiple of num_key_value_heads ({nkv})")
    if getattr(config, "attention_bias", False):
        raise ValueError("attention_bias=True is not supported")
    if getattr(config, "hidden_act", "silu") != "silu":
        raise ValueError("only SwiGLU (hidden_act='silu') is supported")
    rs = getattr(config, "rope_scaling", None)
    if rs is not None and not (isinstance(rs, dict) and rs.get("rope_type", rs.get("type")) == "default"):
        raise ValueError("rope_scaling is not supported (no shipped DreamLLM config enables it)")
    d = config.hidden_size // config.num_attention_heads
    if d not in (64, 128):
        raise ValueError(f"head_dim {d} unsupported (64 or 128)")


# ------------------------------------------------------------------------------------------------ leaf modules
class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        y, rstd, _ = ops.rmsnorm_fwd(x2, weight, eps)
        ctx.save_for_backward(x2, weight, rstd)
        return y.view(shp)

    @staticmethod
    def backward(ctx, dy):
        x2, weight, rstd = ctx.saved_tensors
        dy2 = dy.reshape(x2.shape).contiguous()
        dx, dw = ops.rmsnorm_bwd(dy2, x2, weight, rstd, need_dw=ctx.needs_input_grad[1])
        return dx.view(dy.shape), dw, None


class DreamLLMRMSNorm(nn.Module):
    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, hidden_states):
        return _RMSNormFn.apply(hidden_states, self.weight, self.variance_epsilon)


class RotaryEmbedding(nn.Module):
    """Same buffers as the reference (:97-128): persistent `inv_freq`, non-persistent cos/sin caches built in fp32
    and rounded to the model dtype at use."""

    def __init__(self, dim, max_position_embeddings=2048, base=10000, device=None):
        super().__init__()
        self.dim = dim
        self.max_position_embeddings = max_position_embeddings
        self.base = base
        inv_freq = 1.0 / (self.base ** (torch.arange(0, self.dim, 2).float().to(device) / self.dim))
        self.register_buffer("inv_freq", inv_freq)
        self._set_cos_sin_cache(max_position_embeddings, self.inv_freq.device, torch.get_default_dtype())

    def _set_cos_sin_cache(self, seq_len, device, dtype):
        self.max_seq_len_cached = seq_len
        t = torch.arange(seq_len, device=device, dtype=self.inv_freq.dtype)
        freqs = torch.einsum("i,j->ij", t, self.inv_freq)
        emb = torch.cat((freqs, freqs), dim=-1)
        self.register_buffer("cos_cached", emb.cos().to(dtype), persistent=False)
        self.register_buffer("sin_cached", emb.sin().to(dtype), persistent=False)

    def tables(self, seq_len, device):
        if seq_len > self.max_seq_len_cached:
            self._set_cos_sin_cache(seq_len, device, self.cos_cached.dtype)
        if self.cos_cached.dtype != BF16 or self.cos_cached.device != device:
            self.cos_cached = self.cos_cached.to(device=device, dtype=BF16)
            self.sin_cached = self.sin_cached.to(device=device, dtype=BF16)
        return self.cos_cached, self.sin_cached

    def forward(self, x, seq_len=None):
        cos, sin = self.tables(seq_len, x.device)
        return cos[:seq_len].to(dtype=x.dtype), sin[:seq_len].to(dtype=x.dtype)


def _fuse_rows(params):
    """Make a list of [n_i, K] Parameters contiguous row blocks of one storage (so one GEMM reads them as a single
    [sum n_i, K] weight) without changing their identity / state-dict keys.  Returns the fused view."""
    p0 = params[0]
    esz = p0.element_size()
    ok = all(p.is_contiguous() and p.dtype == p0.dtype and p.device == p0.device for p in params)
    if ok:
        ptr = p0.data_ptr()
        for p in params:
            if p.data_ptr() != ptr or p.untyped_storage().data_ptr() != p0.untyped_storage().data_ptr():
                ok = False
                break
            ptr += p.numel() * esz
    one_d = p0.dim() == 1
    K = 1 if one_d else p0.shape[1]
    rows = sum(p.shape[0] for p in params)
    if not ok:
        fused = torch.empty((rows,) if one_d else (rows, K), dtype=p0.dtype, device=p0.device)
        r = 0
        with torch.no_grad():
            for p in params:
                fused[r:r + p.shape[0]].copy_(p.data)
                p.data = fused[r:r + p.shape[0]]
                r += p.shape[0]
        return fused
    off = p0.storage_offset()
    if one_d:
        return torch.as_strided(p0.data, (rows,), (1,), off)
    return torch.as_strided(p0.data, (rows, K), (K, 1), off)


class DreamLLMMLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.hidden_size = config.hidden_size
        self.intermediate_size = config.intermediate_size
        self.gate_proj = nn.Linear(self.hidden_size, self.intermediate_size, bias=False)
        self.up_proj = nn.Linear(self.hidden_size, self.intermediate_size, bias=False)
        self.down_proj = nn.Linear(self.intermediate_size, self.hidden_size, bias=False)

    def forward(self, x):
        return _MLPFn.apply(x, self.gate_proj.weight, self.up_proj.weight, self.down_proj.weight, self)


class _MLPFn(torch.autograd.Function):
    """Standalone DreamLLMMLP (the decoder layer uses its own fused Function)."""

    @staticmethod
    def forward(ctx, x, wg, wu, wd, mod):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1]).contiguous()
        wgu = _fuse_rows([mod.gate_proj.weight, mod.up_proj.weight])
        gu = ops.linear(x2, wgu)
        act = ops.swiglu_fwd(gu, mod.intermediate_size)
        y = ops.linear(act, wd)
        ctx.save_for_backward(x2, gu, act, wgu, wd)
        ctx.inter = mod.intermediate_size
        return y.view(shp)

    @staticmethod
    def backward(ctx, dy):
        x2, gu, act, wgu, wd = ctx.saved_tensors
        I = ctx.inter
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        dact = ops.linear_dgrad(dy2, wd)
        dwd = ops.linear_wgrad(dy2, act) if ctx.needs_input_grad[3] else None
        dgu = ops.swiglu_bwd(dact, gu, I)
        dx = ops.linear_dgrad(dgu, wgu)
        dwg = dwu = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dwgu = ops.linear_wgrad(dgu, x2)
            dwg, dwu = dwgu[:I], dwgu[I:]
        return dx.view(dy.shape), dwg, dwu, dwd, None


class DreamLLMAttention(nn.Module):
    """Parameter holder with the reference's names; the arithmetic runs inside the fused decoder-layer Function
    (or `forward` below when used standalone)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.hidden_size = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.head_dim = self.hidden_size // self.num_heads
        self.num_key_value_heads = getattr(config, "num_key_value_heads", self.num_heads)
        self.num_key_value_groups = self.num_heads // self.num_key_value_heads
        self.max_position_embeddings = config.max_position_embeddings
        self.rope_theta = getattr(config, "rope_theta", 10000.0)
        if (self.head_dim * self.num_heads) != self.hidden_size:
            raise ValueError(
                f"hidden_size must be divisible by num_heads (got `hidden_size`: {self.hidden_size}"
                f" and `num_heads`: {self.num_heads})."
            )
        self.q_proj = nn.Linear(self.hidden_size, self.num_heads * self.head_dim, bias=False)
        self.k_proj = nn.Linear(self.hidden_size, self.num_key_value_heads * self.head_dim, bias=False)
        self.v_proj = nn.Linear(self.hidden_size, self.num_key_value_heads * self.head_dim, bias=False)
        self.o_proj = nn.Linear(self.num_heads * self.head_dim, self.hidden_size, bias=False)
        self.rotary_emb = RotaryEmbedding(self.head_dim, max_position_embeddings=self.max_position_embeddings,
                                          base=self.rope_theta)
        # q|k|v are row blocks of one fused weight (`_fuse_rows`): under GQA k/v are narrower than q, so the bucket planners cannot glue
        # them by equal shape; this tag keeps each one in the same gradient bucket as the block before it (ddp.plan_runs)
        self.k_proj.weight._dllm_fused_with_prev = True
        self.v_proj.weight._dllm_fused_with_prev = True


DreamLLMFlashAttention2 = DreamLLMAttention  # same kernel either way


# ------------------------------------------------------------------------------------------------ decoder layer
@dataclass
class _LayerMeta:
    num_heads: int
    num_kv_heads: int
    head_dim: int
    inter: int
    eps: float
    B: int
    S: int
    pos: torch.Tensor          # int32 [T]
    cos: torch.Tensor
    sin: torch.Tensor
    seqlens: torch.Tensor | None
    wqkv: torch.Tensor          # fused [(nh + 2 nkv) d, H] view
    wgu: torch.Tensor           # fused [2I, H] view
    p_qkv: tuple = ()           # the Parameters behind the fused views / o_proj / down_proj: their `_dllm_grad_view` (set by a gradient
    p_gu: tuple = ()            # reducer or sharded optimizer) lets the wgrad GEMMs write straight into the flat gradient bucket
    p_o: tuple = ()
    p_d: tuple = ()
    probs: "_AttnProbsSlot | None" = None   # set: also return the attention probabilities (output_attentions)
    cu_seqlens: torch.Tensor | None = None  # set: x is a packed batch [1, T, H]; int32 [n_samples + 1] sample boundaries (device)
    max_seqlen: int = 0                     # packed: the longest sample (host int, sizes the attention grid)


class _AttnProbsSlot:
    """One layer's attention probabilities, materialised at most once per forward.  Non-reentrant gradient checkpointing runs the layer
    forward again inside backward with the same kwargs, so the slot passed there still holds the tensor and the recompute reuses it
    instead of launching the kernel (and allocating B * nh * S * S * 2 bytes) a second time."""
    __slots__ = ("value",)

    def __init__(self):
        self.value = None


def _split_heads(qkv, B, S, nh, nkv, d):
    """q [B,S,nh,d], k and v [B,S,nkv,d]: head-slice views of the fused [B*S, (nh + 2 nkv) d] projection buffer.  Sliced after the
    view so that the token stride stays (nh + 2 nkv) d even when S == 1 (`view` of a slice may give a size-1 dimension any stride)."""
    x = qkv.view(B, S, nh + 2 * nkv, d)
    return x[:, :, :nh], x[:, :, nh:nh + nkv], x[:, :, nh + nkv:]


def _packed_batch(cu_seqlens, max_seqlen, T, device):
    """(cu_seqlens as device int32, max_seqlen as int) of a packed batch of T tokens.  A host `cu_seqlens` (what the collator emits and
    `to_device` leaves on the host) is validated here and uploaded with one small async copy; a device tensor is trusted as the kernels
    trust it, because checking it would cost a device-to-host sync every step."""
    if not torch.is_tensor(cu_seqlens) or cu_seqlens.dim() != 1 or cu_seqlens.numel() < 2:
        raise ValueError("cu_seqlens must be a 1-D tensor [n_samples + 1]")
    if cu_seqlens.is_cuda:
        return cu_seqlens.to(device=device, dtype=torch.int32).contiguous(), int(max_seqlen)
    cu = cu_seqlens.to(torch.int64)
    lens = cu[1:] - cu[:-1]
    if int(cu[0]) != 0 or int(cu[-1]) != T:
        raise ValueError(f"cu_seqlens must run from 0 to the number of packed tokens ({T}), got {int(cu[0])} .. {int(cu[-1])}")
    if bool((lens < 0).any()):
        raise ValueError("cu_seqlens must be non-decreasing")
    longest = int(lens.max())
    if int(max_seqlen) < longest or int(max_seqlen) > T:
        raise ValueError(f"max_seqlen ({max_seqlen}) must bound every sample length (longest {longest}) and not exceed {T}")
    return cu_seqlens.to(torch.int32).to(device, non_blocking=True), int(max_seqlen)


def _packed_positions(cu_seqlens, T):
    """int32 [T] RoPE positions restarting at 0 in every sample, built on the device (`output_size` keeps it free of a host sync)."""
    starts = torch.repeat_interleave(cu_seqlens[:-1], cu_seqlens[1:] - cu_seqlens[:-1], output_size=T)
    return torch.arange(T, device=cu_seqlens.device, dtype=torch.int32) - starts


class _DecoderLayerFn(torch.autograd.Function):
    """One DreamLLMDecoderLayer forward/backward (reference :599-654) as a fixed kernel sequence:

    fwd: rmsnorm -> qkv GEMM -> rope(in place) -> flash-attn -> o GEMM -> (+residual, rmsnorm fused) -> gate|up GEMM
         -> swiglu -> down GEMM -> +residual
    bwd: the transposed sequence; dgrad = NN GEMM, wgrad = TN GEMM, wgrad skipped for frozen weights.
    With `meta.probs` set, forward also returns the attention probabilities [B, nh, S, S] (attn_probs kernel after flash-attn, from its
    lse) as a second, non-differentiable output; y and every gradient are unchanged.
    With `meta.cu_seqlens` set, x is a packed batch [1, T, H] and only the two attention calls differ (variable-length kernels): every
    other kernel of the sequence is token-major and takes its RoPE position per token.
    """

    @staticmethod
    def forward(ctx, x, w_in, wq, wk, wv, wo, w_post, wg, wu, wd, meta: _LayerMeta):
        B, S, H = x.shape
        T = B * S
        nh, nkv, d, I = meta.num_heads, meta.num_kv_heads, meta.head_dim, meta.inter
        x2 = x.reshape(T, H)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        h1, rstd1, _ = ops.rmsnorm_fwd(x2, w_in, meta.eps)
        qkv = ops.linear(h1, meta.wqkv)                                   # [T, (nh + 2 nkv) d]
        ops.rope_(qkv, meta.cos, meta.sin, meta.pos, nh + nkv, d)
        if meta.cu_seqlens is not None:
            ao, lse = ops.attn_fwd_varlen(*(t[0] for t in _split_heads(qkv, 1, T, nh, nkv, d)), meta.cu_seqlens, meta.max_seqlen, causal=True)
        else:
            ao, lse = ops.attn_fwd(*_split_heads(qkv, B, S, nh, nkv, d), causal=True, seqlens=meta.seqlens)
        if meta.probs is not None and meta.probs.value is None:
            meta.probs.value = ops.attn_probs(*_split_heads(qkv, B, S, nh, nkv, d)[:2], lse, causal=True, seqlens=meta.seqlens)
        ao2 = ao.view(T, H)
        o = ops.linear(ao2, wo)
        h2, rstd2, xmid = ops.rmsnorm_fwd(x2, w_post, meta.eps, add=o)    # xmid = x + o
        gu = ops.linear(h2, meta.wgu)                                     # [T, 2I]
        act = ops.swiglu_fwd(gu, I)
        y = ops.linear(act, wd, residual=xmid)                            # down_proj + residual add fused in the GEMM epilogue
        ctx.save_for_backward(x2, w_in, rstd1, h1, qkv, ao2, lse, wo, xmid, w_post, rstd2, h2, gu, act, wd)
        ctx.meta = meta
        if meta.probs is None:
            return y.view(B, S, H)
        ctx.mark_non_differentiable(meta.probs.value)
        return y.view(B, S, H), meta.probs.value

    @staticmethod
    def backward(ctx, dy, *_):
        x2, w_in, rstd1, h1, qkv, ao2, lse, wo, xmid, w_post, rstd2, h2, gu, act, wd = ctx.saved_tensors
        meta = ctx.meta
        B, S, nh, nkv, d, I = meta.B, meta.S, meta.num_heads, meta.num_kv_heads, meta.head_dim, meta.inter
        T, H = x2.shape
        need = ctx.needs_input_grad
        dy2 = dy.reshape(T, H)
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        # ---- MLP
        dact = ops.linear_dgrad(dy2, wd)
        dwd = ops.linear_wgrad(dy2, act, out=grad_out_view(meta.p_d)) if need[9] else None
        dgu = ops.swiglu_bwd(dact, gu, I)
        del dact
        dh2 = ops.linear_dgrad(dgu, meta.wgu)
        dwg = dwu = None
        if need[7] or need[8]:
            dwgu = ops.linear_wgrad(dgu, h2, out=grad_out_view(meta.p_gu))
            dwg, dwu = dwgu[:I], dwgu[I:]
        del dgu
        dxmid, dw_post = ops.rmsnorm_bwd(dh2, xmid, w_post, rstd2, dres=dy2, need_dw=need[6])
        # ---- attention
        dao = ops.linear_dgrad(dxmid, wo)
        dwo = ops.linear_wgrad(dxmid, ao2, out=grad_out_view(meta.p_o)) if need[5] else None
        dqkv = torch.empty_like(qkv)
        if meta.cu_seqlens is not None:
            ops.attn_bwd_varlen(dao, *(t[0] for t in _split_heads(qkv, 1, T, nh, nkv, d)), ao2, lse,
                                *(t[0] for t in _split_heads(dqkv, 1, T, nh, nkv, d)), meta.cu_seqlens, meta.max_seqlen, causal=True)
        else:
            ops.attn_bwd(dao.view(B, S, H), *_split_heads(qkv, B, S, nh, nkv, d), ao2.view(B, S, H), lse,
                         *_split_heads(dqkv, B, S, nh, nkv, d), causal=True, seqlens=meta.seqlens)
        ops.rope_(dqkv, meta.cos, meta.sin, meta.pos, nh + nkv, d, backward=True)
        dh1 = ops.linear_dgrad(dqkv, meta.wqkv)
        dwq = dwk = dwv = None
        if need[2] or need[3] or need[4]:
            dwqkv = ops.linear_wgrad(dqkv, h1, out=grad_out_view(meta.p_qkv))
            dwq, dwk, dwv = dwqkv[:nh * d], dwqkv[nh * d:(nh + nkv) * d], dwqkv[(nh + nkv) * d:]
        dx, dw_in = ops.rmsnorm_bwd(dh1, x2, w_in, rstd1, dres=dxmid, need_dw=need[1])
        return (dx.view(B, S, H) if need[0] else None, dw_in, dwq, dwk, dwv, dwo, dw_post, dwg, dwu, dwd, None)


class KVCache:
    """Preallocated per-layer K/V buffers [B, max_len, num_heads, d] (token-major, read in place by the attention kernel).  Replaces the
    reference's per-layer `torch.cat([past, new], dim=2)` tuples (:444-449); opaque to callers, passed as `past_key_values`.
    `num_heads` is the number of KEY/VALUE heads (`num_key_value_heads`: fewer than the query heads under grouped-query attention)."""

    def __init__(self, num_layers, batch, max_len, num_heads, head_dim, device, dtype=BF16):
        # zero-filled: the attention kernel reads whole 64-row tiles; rows past the valid length are masked in the softmax (p = 0) but
        # still multiply into P.V, so they must be finite (0 * NaN from recycled allocator memory poisoned the output otherwise)
        self.k = [torch.zeros((batch, max_len, num_heads, head_dim), device=device, dtype=dtype) for _ in range(num_layers)]
        self.v = [torch.zeros((batch, max_len, num_heads, head_dim), device=device, dtype=dtype) for _ in range(num_layers)]
        self.len = 0
        self.max_len = max_len
        # key-padding mask of a PADDED prompt batch: uint8 [B, round_up(max_len, 64)], 0 = pad position inside the cache (HF left-pads
        # decoder-only prompts and keeps extending the 2-D attention_mask, reference :1511-1547).  None = no padding anywhere.
        self.mask = None

    def get_seq_length(self):
        return self.len

    def set_mask(self, attention_mask):
        """attention_mask [B, L] (L = tokens in the cache after the current forward), any integer / bool dtype."""
        B, L = attention_mask.shape
        if self.mask is None:
            ld = (self.max_len + 63) // 64 * 64
            self.mask = torch.ones((self.k[0].shape[0], ld), device=self.k[0].device, dtype=torch.uint8)
        if B != self.mask.shape[0] or L > self.mask.shape[1]:
            raise ValueError(f"attention_mask {tuple(attention_mask.shape)} does not fit the kv-cache mask {tuple(self.mask.shape)}")
        self.mask[:, :L] = attention_mask.to(device=self.mask.device, dtype=torch.uint8)

    def repeat_interleave(self, k: int):
        """Beam search: every sample's cache rows repeated k times along the batch dimension.  The buffers are reallocated: build a
        `decode.DecodeGraph` after this call, not before."""
        for li in range(len(self.k)):
            self.k[li] = self.k[li].repeat_interleave(k, dim=0)
            self.v[li] = self.v[li].repeat_interleave(k, dim=0)
        if self.mask is not None:
            self.mask = self.mask.repeat_interleave(k, dim=0).contiguous()
        return self

    def reorder(self, beam_idx):
        """Beam search: row b takes the history of row beam_idx[b] (reference `_reorder_cache`, :1549-1554).  Only the valid prefix
        [:len] is moved.  In place: every buffer keeps its address, so a captured `decode.DecodeGraph` stays valid across a reorder."""
        L = self.len
        for li in range(len(self.k)):
            idx = beam_idx.to(self.k[li].device)
            self.k[li][:, :L] = self.k[li][:, :L].index_select(0, idx)
            self.v[li][:, :L] = self.v[li][:, :L].index_select(0, idx)
        if self.mask is not None:
            self.mask.copy_(self.mask.index_select(0, beam_idx.to(self.mask.device)))
        return self


class DreamLLMDecoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        _check_supported(config)
        self.hidden_size = config.hidden_size
        self.self_attn = DreamLLMAttention(config=config)
        self.mlp = DreamLLMMLP(config)
        self.input_layernorm = DreamLLMRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.post_attention_layernorm = DreamLLMRMSNorm(config.hidden_size, eps=config.rms_norm_eps)

    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None,
                output_attentions=False, use_cache=False, **kwargs):
        """Same contract as the reference (:599-654).  `attention_mask` is the 2-D [B, S] padding mask of the
        flash path (:960-962) or None; right padding as the collator produces (builder_dreamllm.py:467-482).

        `output_attentions=True` returns `(hidden, attn_weights)` (cached path: `(hidden, attn_weights, (cache, layer_idx))`), the
        reference's order.  attn_weights is the post-softmax bf16 [B, nh, q_len, kv_len] of the eager path (:357-378): masked keys 0,
        right-padded query rows a softmax over the sample's valid keys, rows with no visible key uniform 1/kv_len.  It costs
        B * nh * q_len * kv_len * 2 bytes per layer (1.07 GB at B 4, S 2048, 32 heads) and, unlike the reference's, does not require
        grad: no gradient flows back through it.  hidden and every gradient are bit-identical to `output_attentions=False`.

        `cu_seqlens=` (int32 [n_samples + 1]) together with `max_seqlen=` (host int) makes `hidden_states` a packed batch [1, T, H]: the samples' tokens end
        to end, each attending only to itself, positions restarting at 0 in every sample unless `position_ids` says otherwise.  It
        computes what the right-padded batch computes with the pad rows deleted.  Training only: no kv-cache, no `output_attentions`."""
        if not hidden_states.is_cuda:
            raise RuntimeError("DreamLLMDecoderLayer (dreamllm_b200) requires CUDA tensors; there is no CPU fallback")
        if hidden_states.dtype != BF16:
            raise ValueError("dreamllm_b200 computes in bf16: cast the model and inputs with .to(torch.bfloat16)")
        max_seqlen = kwargs.get("max_seqlen")
        cu_seqlens = kwargs.get("cu_seqlens") if max_seqlen is not None else None    # a packed batch is announced by both
        if cu_seqlens is not None:
            if past_key_value is not None or use_cache:
                raise ValueError("a packed batch (cu_seqlens) cannot be combined with a kv-cache (past_key_value / use_cache)")
            if output_attentions:
                raise ValueError("output_attentions is not available for a packed batch (cu_seqlens): the weights are a dense [B, nh, S, S]")
            if hidden_states.shape[0] != 1:
                raise ValueError(f"a packed batch is [1, T, hidden], got {tuple(hidden_states.shape)}")
            cu_seqlens, max_seqlen = _packed_batch(cu_seqlens, max_seqlen, hidden_states.shape[1], hidden_states.device)
        if past_key_value is not None:
            return self._forward_cached(hidden_states, position_ids, past_key_value, output_attentions)
        B, S, H = hidden_states.shape
        if attention_mask is not None and attention_mask.dim() != 2:
            raise ValueError(
                f"Attention mask should be of size {(B, S)} (2-D padding mask, flash path), but is {tuple(attention_mask.size())}")
        att = self.self_attn
        dev = hidden_states.device
        pos = kwargs.get("pos_i32")                       # [B*S] int32, built once per forward by DreamLLMModel._forward
        if pos is None:
            if position_ids is None and cu_seqlens is not None:
                pos = _packed_positions(cu_seqlens, S)
            elif position_ids is None:
                pos = torch.arange(S, device=dev, dtype=torch.int32).repeat(B)
            else:
                pos = position_ids.to(torch.int32).expand(B, S).reshape(-1).contiguous()
        cos, sin = att.rotary_emb.tables(max(S, att.max_position_embeddings), dev)
        seqlens = kwargs.get("seqlens")                   # int32 [B] valid lengths (collator / model loop); else derived from the mask
        if cu_seqlens is not None:
            seqlens = None                                # a packed batch has no pad rows
        elif seqlens is None and attention_mask is not None:
            seqlens = attention_mask.sum(-1).to(torch.int32).contiguous()
        meta = _LayerMeta(att.num_heads, att.num_key_value_heads, att.head_dim, self.mlp.intermediate_size,
                          self.input_layernorm.variance_epsilon, B, S, pos, cos, sin, seqlens,
                          _fuse_rows([att.q_proj.weight, att.k_proj.weight, att.v_proj.weight]),
                          _fuse_rows([self.mlp.gate_proj.weight, self.mlp.up_proj.weight]),
                          (att.q_proj.weight, att.k_proj.weight, att.v_proj.weight), (self.mlp.gate_proj.weight, self.mlp.up_proj.weight),
                          (att.o_proj.weight,), (self.mlp.down_proj.weight,))
        if cu_seqlens is not None:
            meta.cu_seqlens, meta.max_seqlen = cu_seqlens, max_seqlen
        if output_attentions:
            # DreamLLMModel passes its own slot under gradient checkpointing, so that the recompute finds the weights already there
            slot = kwargs.get("attn_probs_slot")
            meta.probs = slot if slot is not None else _AttnProbsSlot()
        outputs = _DecoderLayerFn.apply(hidden_states, self.input_layernorm.weight, att.q_proj.weight, att.k_proj.weight,
                                        att.v_proj.weight, att.o_proj.weight, self.post_attention_layernorm.weight,
                                        self.mlp.gate_proj.weight, self.mlp.up_proj.weight, self.mlp.down_proj.weight, meta)
        if not output_attentions:
            outputs = (outputs,)
        if use_cache:
            raise ValueError("use_cache=True needs a cache: pass past_key_value=(KVCache, layer_idx) (DreamLLMModel does this)")
        return outputs

    @torch.no_grad()
    def _forward_cached(self, hidden_states, position_ids, past_key_value, output_attentions=False):
        """Inference with a kv-cache (prefill or decode; reference :344-355 / :444-449): new keys/values are appended to
        `cache.k/v[layer]` at rows [cache.len, cache.len + S) and attention runs causally (bottom-right aligned) over all of them."""
        cache, li = past_key_value
        B, S, H = hidden_states.shape
        att, mlp = self.self_attn, self.mlp
        nh, nkv, d, I = att.num_heads, att.num_key_value_heads, att.head_dim, mlp.intermediate_size
        start = cache.len
        if start + S > cache.max_len:
            raise ValueError(f"kv-cache overflow: {start} + {S} > {cache.max_len}")
        dev = hidden_states.device
        if position_ids is None:
            pos = torch.arange(start, start + S, device=dev, dtype=torch.int32).repeat(B)
        else:
            pos = position_ids.to(torch.int32).expand(B, S).reshape(-1).contiguous()
        cos, sin = att.rotary_emb.tables(max(start + S, att.max_position_embeddings), dev)
        eps = self.input_layernorm.variance_epsilon
        x2 = hidden_states.reshape(B * S, H).contiguous()
        h1, _, _ = ops.rmsnorm_fwd(x2, self.input_layernorm.weight, eps)
        qkv = ops.linear(h1, _fuse_rows([att.q_proj.weight, att.k_proj.weight, att.v_proj.weight]))
        ops.rope_(qkv, cos, sin, pos, nh + nkv, d)
        q, k, v = _split_heads(qkv, B, S, nh, nkv, d)
        cache.k[li][:, start:start + S].copy_(k)
        cache.v[li][:, start:start + S].copy_(v)
        ao, lse = ops.attn_fwd_cache(q, cache.k[li], cache.v[li], start + S, causal=True, kv_mask=cache.mask, return_lse=True)
        o = ops.linear(ao.view(B * S, H), att.o_proj.weight)
        h2, _, xmid = ops.rmsnorm_fwd(x2, self.post_attention_layernorm.weight, eps, add=o)
        gu = ops.linear(h2, _fuse_rows([mlp.gate_proj.weight, mlp.up_proj.weight]))
        y = ops.linear(ops.swiglu_fwd(gu, I), mlp.down_proj.weight, residual=xmid)
        if output_attentions:
            probs = ops.attn_probs(q, cache.k[li], lse, causal=True, kv_len=start + S, kv_mask=cache.mask)
            return (y.view(B, S, H), probs, (cache, li))
        return (y.view(B, S, H), (cache, li))


# ------------------------------------------------------------------------------------------------ model
class _EmbeddingFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ids, weight, padding_idx=None):
        ctx.save_for_backward(ids, weight)
        ctx.vocab = weight.shape[0]
        ctx.padding_idx = padding_idx
        return ops.embedding_fwd(ids, weight)

    @staticmethod
    def backward(ctx, dy):
        ids, weight = ctx.saved_tensors
        H = dy.shape[-1]
        return None, ops.embedding_bwd(ids, dy.reshape(-1, H).contiguous(), ctx.vocab, out=grad_out_view((weight,)),
                                       padding_idx=ctx.padding_idx), None


class _LMHeadLossFn(torch.autograd.Function):
    """lm_head GEMM + shifted masked-mean CE (reference :1452-1470).  The bf16 logits buffer is overwritten in place
    by dlogits during forward, so nothing of size [T, V] is kept in fp32 and backward is two GEMMs."""

    @staticmethod
    def forward(ctx, h2, weight, shifted_labels):
        logits = ops.linear(h2, weight)                       # [T, V] bf16 (as the reference: bf16 GEMM, then .float())
        loss = ops.cross_entropy_(logits, shifted_labels, 1.0, write_grad=True)
        ctx.save_for_backward(h2, weight, logits)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        h2, weight, dlogits = ctx.saved_tensors
        dh = ops.linear_dgrad(dlogits, weight) if ctx.needs_input_grad[0] else None
        dw = ops.linear_wgrad(dlogits, h2, out=grad_out_view((weight,))) if ctx.needs_input_grad[1] else None
        g = dloss.to(BF16)
        if dh is not None:
            dh.mul_(g)
        if dw is not None:
            dw.mul_(g)
        return dh, dw, None


def average_init_token_embeddings(model, num_added_tokens: int):
    """omni/utils/tokenizer_utils.py:70-80: newly added token rows of embed_tokens / lm_head start at the mean of the existing rows."""
    assert num_added_tokens > 0, "`num_added_tokens` should be positive"
    for emb in (model.get_input_embeddings().weight.data, model.get_output_embeddings().weight.data):
        emb[-num_added_tokens:] = emb[:-num_added_tokens].mean(dim=0, keepdim=True)


@dataclass
class BaseModelOutputWithPast:
    last_hidden_state: torch.Tensor = None
    past_key_values: tuple | None = None
    hidden_states: tuple | None = None
    attentions: tuple | None = None
    additional_log_info: dict | None = None


@dataclass
class CausalLMOutputWithPast:
    loss: torch.Tensor | None = None
    logits: torch.Tensor | None = None
    past_key_values: tuple | None = None
    hidden_states: tuple | None = None
    attentions: tuple | None = None
    additional_log_info: dict | None = None


WEIGHTS_NAME, WEIGHTS_INDEX_NAME = "pytorch_model.bin", "pytorch_model.bin.index.json"
SAFE_WEIGHTS_NAME, SAFE_WEIGHTS_INDEX_NAME = "model.safetensors", "model.safetensors.index.json"


class DreamLLMPreTrainedModel(nn.Module):
    """The slice of `PreTrainedModel` the reference relies on (modeling_dreamllm.py:657-757): class attributes, `_init_weights`,
    `device` / `dtype`, `save_pretrained` / weight loading in the HF on-disk layout (config.json + [sharded] safetensors or .bin), and
    `resize_token_embeddings`.  Not a transformers subclass: the pinned 4.35 API and the installed 5.x one differ, the file format does not."""
    config_class = DreamLLMConfig
    base_model_prefix = "model"
    supports_gradient_checkpointing = True
    _no_split_modules = ["DreamLLMDecoderLayer"]
    _skip_keys_device_placement = "past_key_values"
    _supports_flash_attn_2 = True

    def __init__(self, config=None):
        super().__init__()
        self.config = config
        self._keys_to_ignore_on_save = []           # per instance (the reference's class-level list, :669, is shared between models)

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def gradient_checkpointing_enable(self, gradient_checkpointing_kwargs=None):
        """PreTrainedModel API used by HF Trainer when `gradient_checkpointing=True` (projects/dreamllm/configs/stage1/base.py:90)."""
        for m in self.modules():
            if hasattr(m, "gradient_checkpointing"):
                m.gradient_checkpointing = True

    def gradient_checkpointing_disable(self):
        for m in self.modules():
            if hasattr(m, "gradient_checkpointing"):
                m.gradient_checkpointing = False

    @property
    def is_gradient_checkpointing(self) -> bool:
        return any(getattr(m, "gradient_checkpointing", False) for m in self.modules())

    # ---- HF on-disk layout -------------------------------------------------------------------------------------------------------
    def save_pretrained(self, save_directory: str, max_shard_size: int = 5 * 1024 ** 3, safe_serialization: bool = True):
        """config.json + model weights without the plugin keys (`_keys_to_ignore_on_save`, :826-831, :1230-1235); plugins write their own
        `<save_model_name>.bin` next to them, as DreamLLMTrainer.save_model does (omni/train/dreamllm_trainer.py:104-112)."""
        import json
        import os
        os.makedirs(save_directory, exist_ok=True)
        self.config.save_pretrained(save_directory)
        ignore = set(self._keys_to_ignore_on_save)
        for m in self.modules():
            if m is not self and isinstance(m, DreamLLMPreTrainedModel):
                ignore.update(m._keys_to_ignore_on_save)
        # q|k|v and gate|up are row blocks of one storage: clone so every saved tensor owns its memory
        sd = {k: v.detach().to("cpu").clone().contiguous() for k, v in self.state_dict().items() if k not in ignore}
        shards, cur, cur_bytes = [], {}, 0
        for k, v in sd.items():
            nb = v.numel() * v.element_size()
            if cur and cur_bytes + nb > max_shard_size:
                shards.append(cur)
                cur, cur_bytes = {}, 0
            cur[k] = v
            cur_bytes += nb
        shards.append(cur)
        base, index_name = (SAFE_WEIGHTS_NAME, SAFE_WEIGHTS_INDEX_NAME) if safe_serialization else (WEIGHTS_NAME, WEIGHTS_INDEX_NAME)

        def _write(tensors, fname):
            if safe_serialization:
                from safetensors.torch import save_file
                save_file(tensors, os.path.join(save_directory, fname), metadata={"format": "pt"})
            else:
                torch.save(tensors, os.path.join(save_directory, fname))

        if len(shards) == 1:
            _write(shards[0], base)
        else:
            stem, ext = base.rsplit(".", 1)
            weight_map = {}
            for i, sh in enumerate(shards):
                fname = f"{stem}-{i + 1:05d}-of-{len(shards):05d}.{ext}"
                _write(sh, fname)
                weight_map.update({k: fname for k in sh})
            total = sum(v.numel() * v.element_size() for v in sd.values())
            with open(os.path.join(save_directory, index_name), "w") as f:
                json.dump({"metadata": {"total_size": total}, "weight_map": weight_map}, f, indent=2)
        for _, plugin in self.named_plugins():
            plugin.save_model(save_directory)

    def named_plugins(self):
        cfg = self.config
        out = []
        for name in getattr(cfg, "plugins_init_kwargs", {}) or {}:
            owner = self.model if (cfg.plugins_type[name] == "embedding" and hasattr(self, "model")) else self
            if hasattr(owner, name):
                out.append((name, getattr(owner, name)))
        return out

    @staticmethod
    def _read_checkpoint(path: str) -> dict:
        import json
        import os

        def _load(f):
            if f.endswith(".safetensors"):
                from safetensors.torch import load_file
                return load_file(f)
            return torch.load(f, map_location="cpu", weights_only=True)

        for single, index in ((SAFE_WEIGHTS_NAME, SAFE_WEIGHTS_INDEX_NAME), (WEIGHTS_NAME, WEIGHTS_INDEX_NAME)):
            if os.path.isfile(os.path.join(path, single)):
                return _load(os.path.join(path, single))
            if os.path.isfile(os.path.join(path, index)):
                with open(os.path.join(path, index)) as f:
                    files = sorted(set(json.load(f)["weight_map"].values()))
                sd = {}
                for fn in files:
                    sd.update(_load(os.path.join(path, fn)))
                return sd
        raise OSError(f"no {SAFE_WEIGHTS_NAME} / {WEIGHTS_NAME} (or sharded index) under {path!r}")

    def resize_token_embeddings(self, new_num_tokens: int):
        """PreTrainedModel.resize_token_embeddings as the reference uses it (:1310-1316): grow (or shrink) embed_tokens and lm_head, new
        rows initialised like `_init_weights`."""
        old = self.get_input_embeddings()
        if new_num_tokens == old.weight.shape[0]:
            return old

        def _resized(w, is_embedding):
            new = torch.empty(new_num_tokens, w.shape[1], dtype=w.dtype, device=w.device)
            new.normal_(mean=0.0, std=self.config.initializer_range)
            n = min(new_num_tokens, w.shape[0])
            new[:n] = w.data[:n]
            return new

        emb = nn.Embedding(new_num_tokens, old.weight.shape[1], old.padding_idx, device=old.weight.device, dtype=old.weight.dtype)
        emb.weight.data = _resized(old.weight, True)
        emb.weight.requires_grad_(old.weight.requires_grad)
        self.set_input_embeddings(emb)
        head = self.get_output_embeddings() if hasattr(self, "get_output_embeddings") else None
        if head is not None:
            new_head = nn.Linear(head.weight.shape[1], new_num_tokens, bias=False, device=head.weight.device, dtype=head.weight.dtype)
            new_head.weight.data = _resized(head.weight, False)
            new_head.weight.requires_grad_(head.weight.requires_grad)
            self.set_output_embeddings(new_head)
        self.config.vocab_size = new_num_tokens
        self.vocab_size = new_num_tokens
        if hasattr(self, "model"):
            self.model.vocab_size = new_num_tokens
        return self.get_input_embeddings()

    def _init_weights(self, module):
        std = self.config.initializer_range
        if isinstance(module, nn.Linear):
            module.weight.data.normal_(mean=0.0, std=std)
            if module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.Embedding):
            module.weight.data.normal_(mean=0.0, std=std)
            if module.padding_idx is not None:
                module.weight.data[module.padding_idx].zero_()

    def post_init(self):
        self.apply(self._init_weights)


class DreamLLMModel(DreamLLMPreTrainedModel):
    def __init__(self, config):
        super().__init__(config)
        _check_supported(config)
        self.padding_idx = config.pad_token_id
        self.vocab_size = config.vocab_size
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, self.padding_idx)
        self.layers = nn.ModuleList([DreamLLMDecoderLayer(config) for _ in range(config.num_hidden_layers)])
        self.norm = DreamLLMRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.gradient_checkpointing = False

    def init_plugin_modules(self):
        """reference :822-831: instantiate every "embedding" plugin of `config.plugins_init_kwargs` from its `_target_` string, move it to
        the model's device / dtype, attach it under its registered name, keep its keys out of the LLM checkpoint."""
        for name, init_kwargs in self.config.plugins_init_kwargs.items():
            if self.config.plugins_type[name] == "embedding":
                setattr(self, name, deep_instantiate(init_kwargs).to(self.device, dtype=self.dtype))
                self._keys_to_ignore_on_save.extend(f"model.{name}.{key}" for key in getattr(self, name).state_dict().keys())
        self.attach_plugins()

    def fsdp_ignored_modules(self) -> list:
        """reference :833-838."""
        ignored_modules = []
        for name, _ in self.config.plugins_init_kwargs.items():
            if self.config.plugins_type[name] == "embedding":
                ignored_modules += getattr(self, name).fsdp_ignored_modules()
        return ignored_modules

    def get_input_embeddings(self):
        return self.embed_tokens

    def set_input_embeddings(self, value):
        self.embed_tokens = value

    def _forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None, inputs_embeds=None,
                 use_cache=None, output_attentions=None, output_hidden_states=None, return_dict=None,
                 attention_mask_has_padding=None, seqlens=None, cu_seqlens=None, max_seqlen=None):
        """reference :846-1043.  `attention_mask_has_padding` replaces the `0 in attention_mask` host sync (:962):
        pass False when the collator knows there is no padding (None = decide on the device-free path: keep the
        mask and let the kernel honour seqlens).

        `output_attentions` (None: `config.output_attentions`; forced on by `config.log_attentions`, off by a truthy
        `config._flash_attn_2_enabled`, :920-932) fills `attentions` with one bf16 [B, nh, q_len, kv_len] per layer, B * nh * q_len *
        kv_len * 2 bytes each (1.07 GB per layer at B 4, S 2048, 32 heads); see DreamLLMDecoderLayer.forward.  `config.log_attentions` /
        `config.log_hidden_states` put max |.| of every layer's weights / input (and of the final normed output) into
        `additional_log_info` under the reference's keys (:988-1032), read back with one device-to-host copy per forward.

        `cu_seqlens` with `max_seqlen`: a packed batch, `input_ids` / `inputs_embeds` [1, T] (see DreamLLMDecoderLayer.forward and
        collator.py `pack=True`).  Pass `cu_seqlens` as the collator's host tensor to have it validated without a device read-back.
        `cu_seqlens` without `max_seqlen` is what the collator adds to a right-padded batch for bookkeeping: it changes nothing."""
        cfg = self.config
        if output_attentions is None:
            output_attentions = getattr(cfg, "output_attentions", False)
        log_attentions = getattr(cfg, "log_attentions", False)
        log_hidden_states = getattr(cfg, "log_hidden_states", False)
        if log_attentions:
            output_attentions = True
        if getattr(cfg, "_flash_attn_2_enabled", False) and output_attentions:
            output_attentions = False
            _warn_once("Flash Attention 2.0 is enabled. `output_attentions` is set to `False`.")
        if input_ids is not None and inputs_embeds is not None:
            raise ValueError("You cannot specify both input_ids and inputs_embeds at the same time")
        if input_ids is None and inputs_embeds is None:
            raise ValueError("You have to specify either input_ids or inputs_embeds")
        if inputs_embeds is None:
            inputs_embeds = _EmbeddingFn.apply(input_ids, self.embed_tokens.weight, self.embed_tokens.padding_idx)
        if max_seqlen is None:
            cu_seqlens = None
        if cu_seqlens is not None:
            if use_cache or past_key_values is not None:
                raise ValueError("a packed batch (cu_seqlens) cannot be combined with a kv-cache (past_key_values / use_cache)")
            if output_attentions:
                raise ValueError("output_attentions / log_attentions are not available for a packed batch (cu_seqlens): the weights "
                                 "are a dense [B, nh, S, S]")
            if inputs_embeds.shape[0] != 1:
                raise ValueError(f"a packed batch is one row of T tokens, got batch {inputs_embeds.shape[0]}")
            if attention_mask_has_padding or (attention_mask_has_padding is None and attention_mask is not None
                                              and not bool(attention_mask.all())):
                raise ValueError("a packed batch has no padding: attention_mask must be all ones (or None)")
            cu_seqlens, max_seqlen = _packed_batch(cu_seqlens, max_seqlen, inputs_embeds.shape[1], inputs_embeds.device)
            attention_mask_has_padding = False
        if attention_mask_has_padding is False:
            attention_mask = None
            seqlens = None
        hidden_states = inputs_embeds
        all_hidden = () if output_hidden_states else None
        cache = None
        if use_cache or past_key_values is not None:
            if torch.is_grad_enabled() and hidden_states.requires_grad:
                raise ValueError("kv-cache inference runs under torch.no_grad()")
            B, S, _ = hidden_states.shape
            att = self.layers[0].self_attn
            cache = past_key_values if past_key_values is not None else KVCache(
                len(self.layers), B, self.config.max_position_embeddings, att.num_key_value_heads, att.head_dim, hidden_states.device)
            if attention_mask is not None and attention_mask_has_padding is not False:
                # padded batch inside the cache (reference :960-962 keeps the 2-D mask for the flash path, whose `_upad_input` drops the
                # pad keys; positions come from the mask, :1521-1526).  No host sync: the mask is applied whether or not it has zeros.
                total = cache.len + S
                if attention_mask.dim() != 2 or attention_mask.shape[1] not in (S, total):
                    raise ValueError(f"attention_mask must be [batch, {total}] (cache + new tokens), got {tuple(attention_mask.size())}")
                if attention_mask.shape[1] == S and cache.len > 0:
                    raise ValueError("with a non-empty kv-cache pass the FULL attention_mask (past + new tokens), as HF generate does")
                cache.set_mask(attention_mask)
                if position_ids is None:
                    position_ids = attention_mask.long().cumsum(-1) - 1
                    position_ids = position_ids.masked_fill(attention_mask == 0, 1)[:, -S:]
        pos_i32 = None
        if cache is None:
            # once per forward instead of once per layer: valid lengths for the attention kernels and the int32 RoPE positions
            if attention_mask is not None and seqlens is None:
                if attention_mask.dim() != 2:
                    raise ValueError(f"Attention mask should be 2-D [batch, seq] (flash path), but is {tuple(attention_mask.size())}")
                seqlens = attention_mask.sum(-1).to(torch.int32).contiguous()
            elif seqlens is not None:
                seqlens = seqlens.to(device=hidden_states.device, dtype=torch.int32).contiguous()
            Bq, Sq = hidden_states.shape[:2]
            if position_ids is None and cu_seqlens is not None:
                pos_i32 = _packed_positions(cu_seqlens, Sq)
            elif position_ids is None:
                pos_i32 = torch.arange(Sq, device=hidden_states.device, dtype=torch.int32).repeat(Bq)
            else:
                pos_i32 = position_ids.to(torch.int32).expand(Bq, Sq).reshape(-1).contiguous()
        packed = {} if cu_seqlens is None else {"cu_seqlens": cu_seqlens, "max_seqlen": max_seqlen}
        all_attn = () if output_attentions else None
        logged = []                                       # (key, device scalar) in the reference's order
        for li, layer in enumerate(self.layers):
            if output_hidden_states:
                all_hidden += (hidden_states,)
            if log_hidden_states:
                logged.append((f"hidden_states_layer{li - 1}", hidden_states.detach().abs().max()))
            if cache is not None:
                outs = layer(hidden_states, position_ids=position_ids, past_key_value=(cache, li), use_cache=True,
                             output_attentions=output_attentions)
            elif self.gradient_checkpointing and self.training and torch.is_grad_enabled():
                # reference :994-1003.  Saves only the layer input and re-runs the (deterministic) layer forward inside backward: ~2.15 GB
                # -> 0.27 GB of saved activations per layer at C2 shapes, for one extra forward (+33 % layer FLOPs).  Off by default:
                # 180 GB holds the whole C2 step without recompute (DESIGN.md §3).
                kw = {"output_attentions": True, "attn_probs_slot": _AttnProbsSlot()} if output_attentions else {}
                outs = torch.utils.checkpoint.checkpoint(layer, hidden_states, attention_mask, position_ids, use_reentrant=False,
                                                         seqlens=seqlens, pos_i32=pos_i32, **packed, **kw)
            else:
                outs = layer(hidden_states, attention_mask=attention_mask, position_ids=position_ids, seqlens=seqlens,
                             pos_i32=pos_i32, output_attentions=output_attentions, **packed)
            hidden_states = outs[0]
            if output_attentions:
                all_attn += (outs[1],)
                if log_attentions:
                    logged.append((f"attentions_layer{li}", outs[1].abs().max()))
        if cache is not None:
            cache.len += hidden_states.shape[1]
        hidden_states = self.norm(hidden_states)
        if output_hidden_states:
            all_hidden += (hidden_states,)
        if log_hidden_states:
            logged.append((f"hidden_states_layer{len(self.layers) - 1}", hidden_states.detach().abs().max()))
        info = None
        if logged:                                        # one device-to-host copy instead of the reference's `.cpu().item()` per layer
            values = torch.stack([v.float() for _, v in logged]).tolist()
            info = {k: v for (k, _), v in zip(logged, values)}
        return BaseModelOutputWithPast(last_hidden_state=hidden_states, past_key_values=cache, hidden_states=all_hidden,
                                       attentions=all_attn, additional_log_info=info)

    # ---- plugins (reference :822-831 `init_plugin_modules` instantiates them from config; here they are attached) ----
    def attach_plugins(self, clip_vision_embedding=None, dream_embedding=None, image_start_id=None, dream_start_id=None):
        """Attribute names are the reference's hard-wired ones (:1083, :1093, :1102)."""
        if clip_vision_embedding is not None:
            self.clip_vision_embedding = clip_vision_embedding
        if dream_embedding is not None:
            self.dream_embedding = dream_embedding
        st = getattr(self.config, "special_tokens2ids_dict", None) or None     # {} (the config default) = not populated
        if st is not None:
            image_start_id = st["additional_special_tokens"]["<im_start>"] if image_start_id is None else image_start_id
            dream_start_id = st["additional_special_tokens"]["<dream_start>"] if dream_start_id is None else dream_start_id
        self.image_start_id, self.dream_start_id = image_start_id, dream_start_id
        self.dream_end_id = (st["additional_special_tokens"]["<dream_end>"] if st is not None else
                             (None if dream_start_id is None else dream_start_id + 1))      # token order: tokenization_dreamllm.py:78-94

    def forward(self, input_ids=None, images=None, images_dm=None, attention_mask=None, position_ids=None,
                past_key_values=None, inputs_embeds=None, use_cache=None, output_attentions=None, output_hidden_states=None,
                return_dict=None, attention_mask_has_padding=None, input_ids_cpu=None, splice_plan=None, seqlens=None,
                cu_seqlens=None, max_seqlen=None):
        """reference :1045-1158: embed_tokens -> dream-query splice -> CLIP features -> image splice -> `_forward`.
        `input_ids_cpu` (the collator's host copy) lets the index maps be built without a device->host sync;
        `splice_plan` lets the caller pass prebuilt maps (SURVEY §8f row 3).  Packed batches (`cu_seqlens`, `_forward`): the plan is built
        over the [1, T] ids, where batch-major order is the packed order; that an image or dream-query span stays inside its own sample is
        checked by the collator, which knows the boundaries."""
        # reference :1059-1064: with `freeze_embed_tokens` + newly added special tokens, only the last `num_added_tokens` rows may
        # move — the original rows are restored from the backup every forward (projects/dreamllm/train.py:149-155 sets both attributes)
        backup = getattr(self, "embed_tokens_backup", None)
        if backup is not None:
            with torch.no_grad():
                self.embed_tokens.weight[: -self.num_added_tokens] = backup[: -self.num_added_tokens].data
        need_splice = (images is not None) or (images_dm is not None)
        if past_key_values is not None and images is not None and input_ids is not None and \
                not bool((input_ids == getattr(self, "image_start_id", -1)).any()):
            images = None          # decode steps: do not re-extract CLIP features (reference :1072-1079)
            need_splice = images_dm is not None
        if not need_splice:
            return self._forward(input_ids=input_ids, attention_mask=attention_mask, position_ids=position_ids,
                                 past_key_values=past_key_values, inputs_embeds=inputs_embeds, use_cache=use_cache,
                                 output_attentions=output_attentions, output_hidden_states=output_hidden_states,
                                 attention_mask_has_padding=attention_mask_has_padding, seqlens=seqlens, cu_seqlens=cu_seqlens,
                                 max_seqlen=max_seqlen)
        from .modeling_plugins import build_splice_plan, splice_embeddings
        if input_ids is None:
            raise ValueError("image / dream splicing needs input_ids")
        if inputs_embeds is None:
            inputs_embeds = _EmbeddingFn.apply(input_ids, self.embed_tokens.weight, self.embed_tokens.padding_idx)
        image_features = self.clip_vision_embedding(images) if images is not None else None
        dq = self.dream_embedding.dream_queries if images_dm is not None else None
        if splice_plan is None:
            ids_cpu = input_ids_cpu if input_ids_cpu is not None else input_ids.cpu()
            P = self.clip_vision_embedding.embed_len if images is not None else 0
            Q = self.dream_embedding.embed_len if images_dm is not None else 0
            splice_plan = build_splice_plan(ids_cpu, self.image_start_id if images is not None else -1,
                                            self.dream_start_id if images_dm is not None else -1, P, Q,
                                            0 if images is None else images.shape[0],
                                            None if images_dm is None else images_dm.shape[0], inputs_embeds.device)
        elif splice_plan.device != inputs_embeds.device:       # the collator's host plan: async H2D of a few int32 maps
            splice_plan = splice_plan.to(inputs_embeds.device)
        self._last_splice_plan = splice_plan
        if image_features is not None:
            image_features = image_features.to(inputs_embeds.dtype)
        inputs_embeds = splice_embeddings(inputs_embeds, image_features, dq, splice_plan)
        return self._forward(attention_mask=attention_mask, position_ids=position_ids, inputs_embeds=inputs_embeds,
                             past_key_values=past_key_values, use_cache=use_cache, output_attentions=output_attentions,
                             output_hidden_states=output_hidden_states, attention_mask_has_padding=attention_mask_has_padding,
                             seqlens=seqlens, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen)

    def prepare_dream_queries_with_special_token(self, batch_size: int = 1):
        """reference :1161-1169: embeds of [<dream_start>, dream queries, <dream_end>]."""
        ids = torch.tensor([[self.dream_start_id, self.dream_end_id]], device=self.embed_tokens.weight.device)
        sp = ops.embedding_fwd(ids, self.embed_tokens.weight)
        dq = torch.cat([sp[:, :1], self.dream_embedding().to(sp.dtype), sp[:, 1:]], 1)
        return dq.repeat(batch_size, 1, 1)


class DreamLLMForCausalMLM(DreamLLMPreTrainedModel):
    _tied_weights_keys = {"lm_head.weight": "model.embed_tokens.weight"}

    def __init__(self, config):
        super().__init__(config)
        self.model = DreamLLMModel(config)
        self.vocab_size = config.vocab_size
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.loss_weight_lm = getattr(config, "loss_weight_lm", 1.0)
        self.loss_weight_vm = getattr(config, "loss_weight_vm", 10.0)      # configuration_dreamllm.py:196 default
        self.post_init()

    def init_plugin_modules(self):
        """reference :1224-1235."""
        self.model.init_plugin_modules()
        for name, init_kwargs in self.config.plugins_init_kwargs.items():
            if self.config.plugins_type[name] == "head":
                setattr(self, name, deep_instantiate(init_kwargs).to(self.device, dtype=self.dtype))
                self._keys_to_ignore_on_save.extend(f"{name}.{key}" for key in getattr(self, name).state_dict().keys())

    def fsdp_ignored_modules(self) -> list:
        """reference :1237-1242."""
        ignored_modules = self.model.fsdp_ignored_modules()
        for name, _ in self.config.plugins_init_kwargs.items():
            if self.config.plugins_type[name] == "head":
                ignored_modules += getattr(self, name).fsdp_ignored_modules()
        return ignored_modules

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, tokenizer=None, *model_args, config=None, torch_dtype=None,
                        device=None, reset_plugin_model_name_or_path: bool = False, strict: bool = True, **kwargs):
        """reference :1244-1332: config -> LLM weights -> vocabulary check against the tokenizer -> plugins.  Local directories only (no
        network): HF layout written by `save_pretrained` here, by the reference, or a plain LLaMA / Vicuna export."""
        assert tokenizer is not None, "tokenizer should not be None"
        if not isinstance(config, DreamLLMConfig):
            config_path = config if config is not None else pretrained_model_name_or_path
            config = cls.config_class.from_pretrained(config_path)
        model = cls(config, *model_args)
        sd = cls._read_checkpoint(pretrained_model_name_or_path)
        res = model.load_state_dict(sd, strict=False)
        missing = [k for k in res.missing_keys if not k.endswith("rotary_emb.inv_freq")]      # recomputed buffer (newer LLaMA exports drop it)
        plugin_prefixes = tuple(f"model.{n}." if config.plugins_type[n] == "embedding" else f"{n}." for n in config.plugins_init_kwargs)
        unexpected = [k for k in res.unexpected_keys if not (plugin_prefixes and k.startswith(plugin_prefixes))]
        if strict and (missing or unexpected):
            raise RuntimeError(f"checkpoint does not match the model: missing {missing[:8]}, unexpected {unexpected[:8]}")
        if torch_dtype is not None or device is not None:
            model.to(device=device, dtype=torch_dtype)
        if reset_plugin_model_name_or_path:
            config.reset_plugins_init_kwargs()
        if len(tokenizer) > model.config.vocab_size:                                            # :1310-1316
            model.resize_token_embeddings(len(tokenizer))
        for _, init_kwargs in config.plugins_init_kwargs.items():                               # :1325-1328
            if init_kwargs.get("pretrained_model_name_or_path", None) is None:
                init_kwargs["pretrained_model_name_or_path"] = pretrained_model_name_or_path
        model.init_plugin_modules()                                                             # :1330-1331 (after resize: see the BUG note there)
        return model

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, attention_mask=None, inputs_embeds=None, **kwargs):
        """reference :1511-1547 (the cache is a `KVCache`; a legacy tuple-of-tuples is measured the reference's way)."""
        if past_key_values is not None:
            past_length = past_key_values.get_seq_length() if hasattr(past_key_values, "get_seq_length") else past_key_values[0][0].shape[2]
            if input_ids.shape[1] > past_length:
                remove_prefix_length = past_length
            else:
                remove_prefix_length = input_ids.shape[1] - 1
            input_ids = input_ids[:, remove_prefix_length:]
        position_ids = kwargs.get("position_ids", None)
        if attention_mask is not None and position_ids is None:
            position_ids = attention_mask.long().cumsum(-1) - 1
            position_ids.masked_fill_(attention_mask == 0, 1)
            if past_key_values:
                position_ids = position_ids[:, -input_ids.shape[1]:]
        if inputs_embeds is not None and past_key_values is None:
            model_inputs = {"inputs_embeds": inputs_embeds}
        else:
            model_inputs = {"input_ids": input_ids}
        model_inputs.update({"position_ids": position_ids, "past_key_values": past_key_values, "use_cache": kwargs.get("use_cache"),
                             "attention_mask": attention_mask, "images": kwargs.pop("images", None)})
        return model_inputs

    @staticmethod
    def _reorder_cache(past_key_values, beam_idx):
        """reference :1549-1554; a `KVCache` is reordered in place along its batch dimension."""
        if isinstance(past_key_values, KVCache):
            return past_key_values.reorder(beam_idx)
        reordered_past = ()
        for layer_past in past_key_values:
            reordered_past += (tuple(past_state.index_select(0, beam_idx.to(past_state.device)) for past_state in layer_past),)
        return reordered_past

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def set_input_embeddings(self, value):
        self.model.embed_tokens = value

    def get_output_embeddings(self):
        return self.lm_head

    def set_output_embeddings(self, new_embeddings):
        self.lm_head = new_embeddings

    def set_decoder(self, decoder):
        self.model = decoder

    def get_decoder(self):
        return self.model

    def forward(self, input_ids=None, images=None, images_dm=None, attention_mask=None, position_ids=None,
                past_key_values=None, inputs_embeds=None, labels=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, return_dict=None, attention_mask_has_padding=None, input_ids_cpu=None,
                splice_plan=None, sd_kwargs=None, seqlens=None, shifted_labels=None, cu_seqlens=None, max_seqlen=None, add_time_ids=None,
                **kwargs):
        """reference :1353-1509.  `seqlens` / `shifted_labels` / `splice_plan` / `input_ids_cpu` are the collator's precomputed maps
        (dreamllm_b200/collator.py, SURVEY §8f row 3); without them they are derived here as the reference does.  Comprehension path: images -> CLIP -> splice -> LM loss.  Creation path: dream-query conditioning
        gather (:1401-1418, also returned in `additional_log_info["dream_conditioning"]`) -> optional null-prompt pass (:1420-1439) ->
        `stable_diffusion_head` loss (:1441); `sd_kwargs` forwards injected random draws to the head (tests).
        `cu_seqlens` / `max_seqlen`: a packed batch (`input_ids` / `labels` [1, T], DreamLLMModel._forward); labels derived here get -100
        at the last token of every sample, so that no sample is asked to predict the next one's first token.
        `add_time_ids` [Nd, 6]: the SDXL head's micro-conditioning, one row per dream image (reference modeling_dreamllm_sdxl.py:1357,
        :1440); required when an `StableDiffusionXLHead` is trained, refused for any other head."""
        xl_head = False
        if add_time_ids is not None or images_dm is not None:
            from .modeling_plugins import StableDiffusionXLHead
            xl_head = isinstance(getattr(self, "stable_diffusion_head", None), StableDiffusionXLHead)
        if add_time_ids is not None and not xl_head:
            raise ValueError("add_time_ids is the SDXL head's conditioning; this model's stable_diffusion_head is not a StableDiffusionXLHead")
        if xl_head and self.training and images_dm is not None and add_time_ids is None:
            raise ValueError("training the StableDiffusionXLHead needs add_time_ids [Nd, 6] (the collator emits them from the examples)")
        out = self.model(input_ids=input_ids, images=images, images_dm=images_dm, attention_mask=attention_mask,
                         position_ids=position_ids, past_key_values=past_key_values, inputs_embeds=inputs_embeds,
                         use_cache=use_cache, output_attentions=output_attentions, output_hidden_states=output_hidden_states,
                         attention_mask_has_padding=attention_mask_has_padding, input_ids_cpu=input_ids_cpu,
                         splice_plan=splice_plan, seqlens=seqlens, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen)
        hidden = out.last_hidden_state
        B, S, H = hidden.shape
        h2 = hidden.reshape(B * S, H)
        loss = None
        logits = None
        lm_loss = 0.0
        if labels is not None or shifted_labels is not None:
            if shifted_labels is not None:
                shifted = shifted_labels
            else:
                shifted = torch.full_like(labels, -100)
                shifted[:, :-1] = labels[:, 1:]
                if cu_seqlens is not None and max_seqlen is not None:
                    # (cu[1:] - 1) % T: an empty first sample wraps to the last token, which is -100 already
                    ends = (cu_seqlens[1:].to(shifted.device, non_blocking=True).long() - 1) % shifted.shape[1]
                    shifted[0].index_fill_(0, ends, -100)
            lm_loss = _LMHeadLossFn.apply(h2, self.lm_head.weight, shifted.reshape(-1).contiguous())
            loss = lm_loss * self.loss_weight_lm
        elif kwargs.get("last_token_logits_only", False):
            logits = ops.linear(hidden[:, -1].contiguous(), self.lm_head.weight).view(B, 1, -1).float()
        else:
            logits = ops.linear(h2, self.lm_head.weight).view(B, S, -1).float()
        info = {"lm_loss": lm_loss}
        vm_loss = 0.0
        if images_dm is not None:
            from .modeling_plugins import gather_rows
            plan = self.model._last_splice_plan
            Q = self.model.dream_embedding.embed_len
            enc_h = gather_rows(hidden, plan.cond_rows).view(plan.n_dreams, Q, H)                        # (:1401-1418)
            info["dream_conditioning"] = enc_h
            head = getattr(self, "stable_diffusion_head", None)
            if head is not None and self.training:
                u_enc = None
                if getattr(head, "drop_prob", None) is not None:                                         # (:1420-1439)
                    u_enc = self._null_prompt_states(Q)
                xl = (add_time_ids,) if xl_head else ()
                vm_loss = head(images_dm, enc_h, u_enc, *xl, **(sd_kwargs or {}))   # (:1441) fewer <dream_start> than images_dm -> the head's assert, as the reference
                loss = vm_loss * self.loss_weight_vm + (loss if loss is not None else 0.0)               # (:1486-1488)
        info["vm_loss"] = vm_loss
        sched = getattr(self.config, "loss_scale_schedule", "none")                                   # (:1472-1477, :1489)
        if loss is not None and sched in ("l1_norm", "l2_norm"):
            loss = loss / (self.loss_weight_lm + self.loss_weight_vm if sched == "l1_norm" else
                           math.sqrt(self.loss_weight_lm ** 2 + self.loss_weight_vm ** 2))
        info.update(out.additional_log_info or {})                                                   # (:1494-1500)
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=out.past_key_values, hidden_states=out.hidden_states,
                                      attentions=out.attentions, additional_log_info=info)

    def _null_prompt_states(self, Q):
        """reference :1420-1439: the classifier-free-guidance "null prompt" — an LLM pass over
        [bos, <dream_start>, Q x <im_patch>, <dream_end>, eos] (no `images_dm`, so the patch positions keep their token embeddings) whose
        hidden states at positions [2, 2+Q) replace the conditioning of dropped samples.  Returned as [1, Q, H]; the reference's
        `.repeat(Nd, 1, 1)` is folded into `_CfgDropFn`'s broadcast."""
        from .modeling_plugins import gather_rows
        m = self.model
        st = getattr(self.config, "special_tokens2ids_dict", None) or None     # {} (the config default) = not populated
        if st is not None:
            patch_id = st["additional_special_tokens"]["<im_patch>"]
            bos_id, eos_id = st["<s>"], st["</s>"]                  # DEFAULT_BOS/EOS_TOKEN keys (:1396-1397)
        else:                                                           # token order: tokenization_dreamllm.py:78-94
            patch_id, bos_id, eos_id = m.dream_start_id - 4, self.config.bos_token_id, self.config.eos_token_id
        dev = m.embed_tokens.weight.device
        ids = torch.tensor([[bos_id, m.dream_start_id] + [patch_id] * Q + [m.dream_end_id, eos_id]], device=dev)
        u_hidden = m(input_ids=ids, attention_mask_has_padding=False).last_hidden_state                  # [1, Q+4, H]
        rows = torch.arange(2, 2 + Q, device=dev, dtype=torch.int32)
        return gather_rows(u_hidden, rows).view(1, Q, u_hidden.shape[-1])

    # ---------------------------------------------------------------------------------------------- inference entry points
    @torch.no_grad()
    def generate(self, input_ids, images=None, max_new_tokens=16, do_sample=False, temperature=1.0, top_k=0, top_p=1.0,
                 repetition_penalty=1.0, eos_token_id=None, pad_token_id=None, generator=None, attention_mask=None,
                 stopping_criteria=None, use_cuda_graph=False, **kwargs):
        """Decoding with the kv-cache (what HF `generate` does through the reference: omni/eval/vqa/vqa_inference.py:112-130): greedy or
        temperature / top-k / top-p sampling with HF's processor semantics, or beam search with `num_beams > 1` (dreamllm_b200/generation.py).
        `use_cuda_graph=True` replays each decode step from one captured CUDA graph (dreamllm_b200/decode.py)."""
        from .generation import beam_search, generate
        num_beams = int(kwargs.get("num_beams", 1))
        if num_beams > 1:                                      # the reference's default VQA eval: num_beams=5 (vqa_inference.py:111-119)
            if do_sample:
                raise NotImplementedError("beam sampling (num_beams > 1 with do_sample=True) is not built")
            if attention_mask is not None and not bool(attention_mask.all()) and not bool(attention_mask[:, -1].all()):
                if images is not None:
                    raise NotImplementedError("right-padded prompt batches with images: left-pad them or pass the prompts one at a time")
                from .generation import ragged
                kw = dict(kwargs)
                return ragged(lambda ids: self.generate(ids, max_new_tokens=max_new_tokens, eos_token_id=eos_token_id, pad_token_id=pad_token_id,
                                                        stopping_criteria=stopping_criteria, use_cuda_graph=use_cuda_graph, **kw),
                              input_ids, attention_mask,
                              pad_token_id if pad_token_id is not None else (eos_token_id if isinstance(eos_token_id, int) else 0))
            return beam_search(self, input_ids, images=images, num_beams=num_beams, max_new_tokens=max_new_tokens,
                               length_penalty=kwargs.get("length_penalty", 1.0), early_stopping=kwargs.get("early_stopping", False),
                               eos_token_id=eos_token_id, pad_token_id=pad_token_id, stopping_criteria=stopping_criteria,
                               length_normalization=kwargs.get("length_normalization", "generated"), attention_mask=attention_mask,
                               use_cuda_graph=use_cuda_graph)
        return generate(self, input_ids, images=images, max_new_tokens=max_new_tokens, do_sample=do_sample, temperature=temperature,
                        top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty, eos_token_id=eos_token_id,
                        pad_token_id=pad_token_id, generator=generator, attention_mask=attention_mask,
                        stopping_criteria=stopping_criteria, use_cuda_graph=use_cuda_graph)

    @torch.no_grad()
    def generate_greedy(self, input_ids, max_new_tokens=16, images=None, eos_token_id=None):
        """Greedy decoding (`do_sample=False`): token-id / argmax path, bit-exact w.r.t. a full re-forward."""
        return self.generate(input_ids, images=images, max_new_tokens=max_new_tokens, do_sample=False, eos_token_id=eos_token_id)

    @torch.no_grad()
    def get_prompt_embeds(self, input_ids, images=None):
        """reference :1598-1673 (token ids in; the tokenizer is out of scope): LLM pass 1 over the prompt with use_cache, pass 2 over
        [<dream_start>, dream queries, <dream_end>] against the cache; returns last hidden states [:, 1:-1] = [B, Q, H]."""
        text_out = self(input_ids=input_ids, images=images, use_cache=True, last_token_logits_only=True)
        dq = self.model.prepare_dream_queries_with_special_token(batch_size=input_ids.shape[0])
        out = self(inputs_embeds=dq, past_key_values=text_out.past_key_values, use_cache=True, output_hidden_states=True,
                   last_token_logits_only=True)
        return out.hidden_states[-1][:, 1:-1, :]

    @torch.no_grad()
    def stable_diffusion_pipeline(self, input_ids, negative_input_ids=None, images=None, guidance_scale=7.5, num_inference_steps=50,
                                  height=None, width=None, latents=None, generator=None, output_type="latent", scheduler="ddpm",
                                  use_cuda_graph=True):
        """reference :1765-1889: encode_prompt (two kv-cache LLM passes, also for the negative prompt) -> StableDiffusionHead.pipeline."""
        prompt_embeds = self.get_prompt_embeds(input_ids, images)
        negative = None
        if guidance_scale > 1.0:
            if negative_input_ids is None:
                raise ValueError("classifier-free guidance needs negative_input_ids (the reference's default negative prompt is text)")
            negative = self.get_prompt_embeds(negative_input_ids)
        return self.stable_diffusion_head.pipeline(height=height, width=width, num_inference_steps=num_inference_steps,
                                                   guidance_scale=guidance_scale, generator=generator, latents=latents,
                                                   prompt_embeds=prompt_embeds, negative_prompt_embeds=negative, output_type=output_type,
                                                   scheduler=scheduler, use_cuda_graph=use_cuda_graph)

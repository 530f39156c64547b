"""One decode token as one captured CUDA graph (`generate(..., use_cuda_graph=True)`).

The eager cached decode (`DreamLLMDecoderLayer._forward_cached`) needs host values every token: the cache offset for the K/V copies and
the attention's loop bounds.  `DecodeGraph` keeps them on the device instead — positions [B] and the cache length are int32 device
counters that the step itself advances — so the whole step (embedding, every layer, final norm, lm_head) is position-independent and is
recorded once and replayed for every token:

    per layer: rmsnorm -> qkv GEMM -> rope_append_kv (RoPE of q/k + k/v written to cache row kv_len) -> attn_decode (split-KV)
               -> o GEMM -> rmsnorm(+residual) -> gate|up GEMM -> swiglu -> down GEMM(+residual)

The GEMMs, norms and swiglu are the eager path's launches with the same shapes, so they compute the same bits; `attn_decode` sums in a
different order from `attn_fwd_cache`, which is why the graph path is opt-in.  Token selection stays outside the graph.
"""
from __future__ import annotations

import torch

from . import ops


def _cache_key(cache, B):
    return (tuple(t.data_ptr() for t in cache.k), tuple(t.data_ptr() for t in cache.v),
            None if cache.mask is None else cache.mask.data_ptr(), B)


class DecodeGraph:
    """Static buffers and the captured decode step of `model` (a DreamLLMForCausalMLM) over `cache` (a KVCache holding B rows).

    `ids` [B] int64: the tokens to feed (write them with `ids.copy_(...)`); `logits` [B, V] fp32: the next-token logits after a step.
    `positions` (int [B] tensor, default: every row at `cache.len`): the RoPE position of the first token fed; left-padded batches pass
    the number of real prompt tokens of each row.  Every step advances the positions, the device cache length and `cache.len` by one.

    The graph holds the cache's tensors by address: it is valid while those tensors live, so `KVCache.repeat_interleave` (which
    reallocates) must run before the DecodeGraph is built, while `KVCache.reorder` (in place) may run between replays."""

    def __init__(self, model, cache, B, positions=None):
        from .generation import check_graph_decode
        check_graph_decode(model)
        if cache.k[0].shape[0] != B:
            raise ValueError(f"the kv-cache holds {cache.k[0].shape[0]} rows, not B = {B}")
        self.model, self.cache, self.B = model, cache, B
        m = model.model
        dev = cache.k[0].device
        att = m.layers[0].self_attn
        self.nh, self.nkv, self.d = att.num_heads, att.num_key_value_heads, att.head_dim
        # reference :1059-1064 restores the frozen embedding rows every forward; the rows do not change during decoding, so once is enough
        backup = getattr(m, "embed_tokens_backup", None)
        if backup is not None:
            with torch.no_grad():
                m.embed_tokens.weight[: -m.num_added_tokens] = backup[: -m.num_added_tokens].data
        from .modeling_dreamllm import _fuse_rows
        self.layers = []
        for layer in m.layers:
            a, mlp = layer.self_attn, layer.mlp
            self.layers.append((layer.input_layernorm.weight, _fuse_rows([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight]),
                                a.o_proj.weight, layer.post_attention_layernorm.weight,
                                _fuse_rows([mlp.gate_proj.weight, mlp.up_proj.weight]), mlp.down_proj.weight, mlp.intermediate_size,
                                layer.input_layernorm.variance_epsilon))
        self.cos, self.sin = att.rotary_emb.tables(max(cache.max_len, att.max_position_embeddings), dev)
        self.ids = torch.zeros(B, dtype=torch.long, device=dev)
        if positions is None:
            self.pos = torch.full((B,), cache.len, dtype=torch.int32, device=dev)
        else:
            self.pos = positions.to(device=dev, dtype=torch.int32).reshape(B).clone()
        self.lens = torch.tensor([cache.len, cache.len + 1], dtype=torch.int32, device=dev)   # [row written this step, rows attended]
        self.workspace = torch.empty(ops.attn_decode_workspace_bytes(B, self.nh, self.nkv, self.d, cache.max_len), dtype=torch.uint8,
                                     device=dev)
        self.logits = torch.empty((B, model.lm_head.weight.shape[0]), dtype=torch.float32, device=dev)
        self.graph = None
        self._key = _cache_key(cache, B)

    def _step(self):
        m, cache = self.model.model, self.cache
        nh, nkv, d = self.nh, self.nkv, self.d
        x = ops.embedding_fwd(self.ids, m.embed_tokens.weight)                                  # [B, H]
        for li, (w_in, wqkv, wo, w_post, wgu, wd, inter, eps) in enumerate(self.layers):
            h1, _, _ = ops.rmsnorm_fwd(x, w_in, eps)
            qkv = ops.linear(h1, wqkv)                                                          # [B, (nh + 2 nkv) d]
            ops.rope_append_kv_(qkv, self.cos, self.sin, self.pos, cache.k[li], cache.v[li], self.lens[0:1], nh, nkv, d)
            ao = ops.attn_decode(qkv[:, :nh * d].view(self.B, nh, d), cache.k[li], cache.v[li], self.lens[1:2], kv_mask=cache.mask,
                                 workspace=self.workspace)
            o = ops.linear(ao, wo)
            h2, _, xmid = ops.rmsnorm_fwd(x, w_post, eps, add=o)
            gu = ops.linear(h2, wgu)
            x = ops.linear(ops.swiglu_fwd(gu, inter), wd, residual=xmid)
        h, _, _ = ops.rmsnorm_fwd(x, m.norm.weight, m.norm.variance_epsilon)
        self.logits.copy_(ops.linear(h, self.model.lm_head.weight))
        self.lens += 1
        self.pos += 1

    def _check(self):
        if _cache_key(self.cache, self.B) != self._key:
            raise RuntimeError("the kv-cache tensors changed since this DecodeGraph was built (e.g. KVCache.repeat_interleave): build a "
                               "new DecodeGraph")
        if self.cache.len + 1 > self.cache.max_len:
            raise ValueError(f"kv-cache overflow: {self.cache.len} + 1 > {self.cache.max_len}")

    @torch.no_grad()
    def step(self):
        """One decode step, run eagerly."""
        self._check()
        self._step()
        self.cache.len += 1
        return self.logits

    @torch.no_grad()
    def capture(self):
        """Record the step once.  A warm-up step runs first on a side stream (module loading, one-time kernel attributes); it writes the
        cache row the next step overwrites, and the counters it advanced are rewound."""
        self._check()
        lens0, pos0 = self.lens.clone(), self.pos.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self._step()
        torch.cuda.current_stream().wait_stream(s)
        self.lens.copy_(lens0)
        self.pos.copy_(pos0)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._step()
        self.graph = graph
        return self

    @torch.no_grad()
    def replay(self):
        """One decode step from the captured graph (captured on first use)."""
        if self.graph is None:
            self.capture()
        self._check()
        self.graph.replay()
        self.cache.len += 1
        return self.logits

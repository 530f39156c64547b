"""Mint the grouped-query attention goldens from the REFERENCE'S OWN CODE (needs a checkout of the reference).

    python -m oracle.gen_golden_gqa [case ...]

The reference's DreamLLMDecoderLayer (exec'd verbatim by oracle/ref_exec.py) with num_key_value_heads < num_attention_heads: k_proj /
v_proj narrower than q_proj, keys / values repeated to the query heads by `repeat_kv` (modeling_dreamllm.py:242-252, :357-358).
Files (names deliberately outside the `decoder_layer_*.npz` pattern, which the multi-head tests glob):

  * tests/golden/gqa_layer_<case>.npz — fp32 forward + backward of one layer, the layout of oracle/gen_golden.py plus `kv_heads`,
    `rope_theta` and the reference layer's state-dict names / shapes.  y / dx are always stored strided (`stride` = row step, column
    step) and `y_abs_sum` / `dx_abs_sum` are whole-tensor sums over the valid (non-pad) rows, so every file stays under 1 MB;
  * tests/golden/gqa_kvcache_layer.npz — the left-padded prefill + decode scenario of gqa_oracle.cached_decode_scenario, 8 / 2 heads;
  * tests/golden/gqa_bf16_pins.npz — the reference layer run in bf16 (one causal forward, and the kv-cache scenario), raw bf16 bits.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gqa_oracle as G  # noqa: E402
from oracle import gen_golden, ref_exec  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
BF = torch.bfloat16

CASES = {
    # name: (hidden, inter, heads, kv_heads, bsz, seq, seed, pad (right-pad tokens of sample 1), rope_theta, (row step, column step))
    "g4d64": (512, 1024, 8, 2, 2, 200, 31, 0, 10000.0, (2, 2)),
    "ragged": (1024, 2048, 8, 4, 2, 160, 32, 77, 10000.0, (1, 4)),
    "mqa": (512, 1024, 4, 1, 2, 128, 33, 0, 10000.0, (2, 2)),
    # Llama-3-8B layer: hidden 4096, inter 14336, 32 / 8 heads, rope_theta 500000
    "l3": (4096, 14336, 32, 8, 1, 512, 34, 0, 500000.0, (4, 8)),
}
KV_CASE = (512, 1024, 8, 2)                       # hidden, inter, heads, kv_heads of the kv-cache scenario
BF16_LAYER_CASE = (512, 1024, 8, 2, 2, 40, 5)     # hidden, inter, heads, kv_heads, bsz, seq, seed


def pad_mask(bsz, seq, pad):
    if not pad:
        return None
    am = torch.ones(bsz, seq, dtype=torch.long)
    am[1, seq - pad:] = 0
    return am


def reference_layer(ns, hidden, inter, heads, kv_heads, params, rope_theta=10000.0):
    cfg = ref_exec.make_config(hidden, inter, heads, rope_theta=rope_theta)
    cfg.num_key_value_heads = kv_heads
    layer = ns["DreamLLMDecoderLayer"](cfg).float()
    sd = {k: v.clone() for k, v in params.items()}
    sd["self_attn.rotary_emb.inv_freq"] = layer.self_attn.rotary_emb.inv_freq.clone()
    layer.load_state_dict(sd)
    return layer


def run_layer_case(ns, name):
    hidden, inter, heads, kv_heads, bsz, seq, seed, pad, theta, (rs, cs) = CASES[name]
    p = G.init_layer_params(hidden, inter, seed, heads, kv_heads)
    layer = reference_layer(ns, hidden, inter, heads, kv_heads, p, theta)
    x, gy = gen_golden.make_inputs(hidden, bsz, seq, seed)
    x.requires_grad_(True)
    am = pad_mask(bsz, seq, pad)
    mask = ref_exec.causal_mask_4d(bsz, seq, torch.float32, am)
    pos = torch.arange(seq)[None].expand(bsz, -1)
    y = layer(x, attention_mask=mask, position_ids=pos)[0]
    valid = torch.ones(bsz, seq, dtype=torch.bool)
    if am is not None:
        gy = gy * am[..., None]                   # padded positions carry no loss (labels are -100 there)
        valid = am.bool()
    y.backward(gy)
    sd = layer.state_dict()
    out = {
        "shape": np.array([hidden, inter, heads, bsz, seq, seed, pad], dtype=np.int64),
        "kv_heads": np.int64(kv_heads),
        "rope_theta": np.float64(theta),
        "x_checksum": np.float64(gen_golden.checksum(x.detach())),
        "w_checksum": np.float64(sum(gen_golden.checksum(v) for v in p.values())),
        "stride": np.array([rs, cs], dtype=np.int64),
        "y": y.detach()[:, ::rs, ::cs].numpy().astype(np.float32),
        "dx": x.grad[:, ::rs, ::cs].numpy().astype(np.float32),
        "y_abs_sum": np.float64(gen_golden.checksum(y.detach()[valid])),
        "dx_abs_sum": np.float64(gen_golden.checksum(x.grad[valid])),
        "sd_names": np.array(list(sd.keys())),
        "sd_shapes": np.array([list(v.shape) + [0] * (2 - v.dim()) for v in sd.values()], dtype=np.int64),
    }
    for k, prm in layer.named_parameters():
        g = prm.grad
        out["d_" + k] = (g[:8, :64] if g.dim() == 2 else g).numpy().astype(np.float32)
        out["dsum_" + k] = np.float64(g.double().sum())
    return out


def run_cached(ns, dtype=torch.float32):
    """The reference layer driven with `past_key_value` / `use_cache=True` over cached_decode_scenario (left-padded batch, prefill +
    single-token steps, 4-D masks from the reference's own `_prepare_4d_causal_attention_mask`).  Returns the outputs of every call."""
    from transformers.modeling_attn_mask_utils import _prepare_4d_causal_attention_mask
    hidden, inter, heads, kv_heads = KV_CASE
    p, calls = G.cached_decode_scenario(hidden, inter, heads, kv_heads)
    layer = reference_layer(ns, hidden, inter, heads, kv_heads, p).to(dtype)
    past, ys = None, []
    with torch.no_grad():
        for x, am, pos in calls:
            past_len = 0 if past is None else past[0].shape[2]
            mask = _prepare_4d_causal_attention_mask(am, (x.shape[0], x.shape[1]), x.to(dtype), past_len)
            y, past = layer(x.to(dtype), attention_mask=mask, position_ids=pos, past_key_value=past, use_cache=True)
            ys.append(y)
    return calls, ys, past


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().to(BF).contiguous().view(torch.int16).numpy().view(np.uint16)


def _save(name, out):
    path = os.path.join(OUT, name)
    np.savez_compressed(path, **out)
    size = os.path.getsize(path)
    assert size < 1 << 20, (path, size)
    print(path, size // 1024, "KiB")


def main():
    assert ref_exec.available(), "needs a checkout of the reference"
    torch.set_num_threads(8)
    ns = ref_exec.load_reference_namespace()
    only = set(sys.argv[1:])
    for name in CASES:
        if not only or name in only:
            _save(f"gqa_layer_{name}.npz", run_layer_case(ns, name))
    if not only or "kvcache" in only:
        calls, ys, past = run_cached(ns)
        out = {"shape": np.array(KV_CASE, dtype=np.int64), "k_final": past[0][:, :, -4:].numpy().astype(np.float32)}
        for i, ((x, am, pos), y) in enumerate(zip(calls, ys)):
            out[f"y{i}"] = y.numpy().astype(np.float32)
            out[f"mask{i}"] = am.numpy()
        _save("gqa_kvcache_layer.npz", out)
    if not only or "bf16" in only:
        hidden, inter, heads, kv_heads, bsz, seq, seed = BF16_LAYER_CASE
        layer = reference_layer(ns, hidden, inter, heads, kv_heads, G.init_layer_params(hidden, inter, seed, heads, kv_heads)).to(BF)
        x, _ = gen_golden.make_inputs(hidden, bsz, seq, seed)
        pos = torch.arange(seq)[None].expand(bsz, -1)
        out = {}
        with torch.no_grad():
            out["layer_y"] = _bits(layer(x.to(BF), attention_mask=ref_exec.causal_mask_4d(bsz, seq, BF), position_ids=pos)[0])
        _, ys, _ = run_cached(ns, BF)
        for i, y in enumerate(ys):
            out[f"kv_y{i}"] = _bits(y)
        _save("gqa_bf16_pins.npz", out)


if __name__ == "__main__":
    main()

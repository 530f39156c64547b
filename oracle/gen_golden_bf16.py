"""Mint tests/golden/bf16_pins.npz from the reference's own DreamLLMDecoderLayer run in bf16 (needs a checkout of the reference).

    python -m oracle.gen_golden_bf16

Two scenarios, both at hidden 256 / 2 heads, stored as the raw bf16 bits (uint16):
  * `layer_y`: one causal forward over 2 x 40 tokens (the inputs of oracle.gen_golden.make_inputs, seed 5);
  * `kv_y{i}`: the left-padded kv-cache scenario of oracle.decoder_oracle.cached_decode_scenario (prefill + 3 single-token steps) driven
    through the reference's `past_key_value` / `use_cache=True` path.
tests/test_oracle_pin.py checks that the oracle run in bf16 shares the reference's rounding points against these outputs.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import decoder_oracle as O
from oracle import gen_golden, ref_exec

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "bf16_pins.npz")
BF = torch.bfloat16
LAYER_CASE = (256, 512, 2, 2, 40, 5)      # hidden, inter, heads, bsz, seq, seed
KV_CASE = (256, 512, 2)                   # hidden, inter, heads


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().to(BF).contiguous().view(torch.int16).numpy().view(np.uint16)


def _reference_layer(ns, hidden, inter, heads, params):
    layer = ns["DreamLLMDecoderLayer"](ref_exec.make_config(hidden, inter, heads)).float()
    sd = {k: v.clone() for k, v in params.items()}
    sd["self_attn.rotary_emb.inv_freq"] = layer.self_attn.rotary_emb.inv_freq.clone()
    layer.load_state_dict(sd)
    return layer.to(BF)


def main() -> None:
    assert ref_exec.available(), "needs a checkout of the reference"
    from transformers.modeling_attn_mask_utils import _prepare_4d_causal_attention_mask
    ns = ref_exec.load_reference_namespace()
    out = {}
    hidden, inter, heads, bsz, seq, seed = LAYER_CASE
    layer = _reference_layer(ns, hidden, inter, heads, O.init_layer_params(hidden, inter, seed))
    x, _ = gen_golden.make_inputs(hidden, bsz, seq, seed)
    pos = torch.arange(seq)[None].expand(bsz, -1)
    with torch.no_grad():
        out["layer_y"] = _bits(layer(x.to(BF), attention_mask=ref_exec.causal_mask_4d(bsz, seq, BF), position_ids=pos)[0])
    hidden, inter, heads = KV_CASE
    p, calls = O.cached_decode_scenario(hidden, inter, heads)
    layer = _reference_layer(ns, hidden, inter, heads, p)
    past = None
    with torch.no_grad():
        for i, (x, am, pos) in enumerate(calls):
            past_len = 0 if past is None else past[0].shape[2]
            mask = _prepare_4d_causal_attention_mask(am, (x.shape[0], x.shape[1]), x.to(BF), past_len)
            yr, past = layer(x.to(BF), attention_mask=mask, position_ids=pos, past_key_value=past, use_cache=True)
            out[f"kv_y{i}"] = _bits(yr)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()

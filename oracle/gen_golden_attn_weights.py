"""Mint the attention-weight goldens from the REFERENCE'S OWN CODE (needs a checkout of the reference).

    python -m oracle.gen_golden_attn_weights [case ...]

The reference's DreamLLMDecoderLayer (exec'd verbatim by oracle/ref_exec.py) called with `output_attentions=True`: its second output is
the eager path's post-softmax weights (modeling_dreamllm.py:357-378).  Each file holds the fp32 run's weights (`w*`) and the bf16 run's
as raw bf16 bits (`w*_bf16`), all under 1 MB:

  * tests/golden/attn_weights_<case>.npz — one causal layer forward with the 4-D mask `_prepare_4d_causal_attention_mask` builds from the
    2-D padding mask `mask`:
      - g4d64: grouped-query (8 / 2 heads, d 64), sample 1 right-padded, sample 2 of length 0 (every row uniform);
      - mha128: multi-head, d 128;
  * tests/golden/attn_weights_kvcache.npz — the left-padded prefill + 3 single-token steps of gqa_oracle.cached_decode_scenario (8 / 2
    heads), `past_key_value` / `use_cache=True`: `w{i}` is call i's [B, nh, S_i, past_i + S_i], `mask{i}` its 2-D mask.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gqa_oracle as G  # noqa: E402
from oracle import gen_golden, gen_golden_gqa, ref_exec  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
BF = torch.bfloat16

CASES = {
    # name: (hidden, inter, heads, kv_heads, seed, valid length of each sample (sequence length = the first))
    "g4d64": (512, 1024, 8, 2, 41, (72, 45, 0)),
    "mha128": (512, 1024, 4, 4, 42, (80, 80)),
}
KV_CASE = (512, 1024, 8, 2)                       # hidden, inter, heads, kv_heads of the kv-cache scenario


def length_mask(lens):
    """2-D right-padding mask [B, lens[0]]: sample b has lens[b] valid tokens."""
    am = torch.zeros(len(lens), lens[0], dtype=torch.long)
    for b, n in enumerate(lens):
        am[b, :n] = 1
    return am


def layer_case(name):
    """(params, x, 2-D mask, position ids) of a layer case, drawn as oracle/gen_golden_gqa.py draws its inputs."""
    hidden, inter, heads, kv_heads, seed, lens = CASES[name]
    p = G.init_layer_params(hidden, inter, seed, heads, kv_heads)
    x, _ = gen_golden.make_inputs(hidden, len(lens), lens[0], seed)
    return p, x, length_mask(lens), torch.arange(lens[0])[None].expand(len(lens), -1)


def run_layer_case(ns, name, dtype):
    hidden, inter, heads, kv_heads, _, lens = CASES[name]
    p, x, am, pos = layer_case(name)
    layer = gen_golden_gqa.reference_layer(ns, hidden, inter, heads, kv_heads, p).to(dtype)
    with torch.no_grad():
        _, w = layer(x.to(dtype), attention_mask=ref_exec.causal_mask_4d(len(lens), lens[0], dtype, am), position_ids=pos,
                     output_attentions=True)
    return w, am


def run_cached(ns, dtype):
    from transformers.modeling_attn_mask_utils import _prepare_4d_causal_attention_mask
    hidden, inter, heads, kv_heads = KV_CASE
    p, calls = G.cached_decode_scenario(hidden, inter, heads, kv_heads)
    layer = gen_golden_gqa.reference_layer(ns, hidden, inter, heads, kv_heads, p).to(dtype)
    past, ws = None, []
    with torch.no_grad():
        for x, am, pos in calls:
            past_len = 0 if past is None else past[0].shape[2]
            mask = _prepare_4d_causal_attention_mask(am, (x.shape[0], x.shape[1]), x.to(dtype), past_len)
            _, w, past = layer(x.to(dtype), attention_mask=mask, position_ids=pos, past_key_value=past, output_attentions=True,
                               use_cache=True)
            ws.append(w)
    return calls, ws


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().to(BF).contiguous().view(torch.int16).numpy().view(np.uint16)


def main():
    assert ref_exec.available(), "needs a checkout of the reference"
    torch.set_num_threads(8)
    ns = ref_exec.load_reference_namespace()
    only = set(sys.argv[1:])
    for name in CASES:
        if not only or name in only:
            w, am = run_layer_case(ns, name, torch.float32)
            wb, _ = run_layer_case(ns, name, BF)
            gen_golden_gqa._save(f"attn_weights_{name}.npz", {"mask": am.numpy(), "w": w.numpy().astype(np.float32), "w_bf16": _bits(wb)})
    if not only or "kvcache" in only:
        calls, ws = run_cached(ns, torch.float32)
        _, wbs = run_cached(ns, BF)
        out = {"shape": np.array(KV_CASE, dtype=np.int64)}
        for i, ((_, am, _), w, wb) in enumerate(zip(calls, ws, wbs)):
            out[f"w{i}"] = w.numpy().astype(np.float32)
            out[f"w{i}_bf16"] = _bits(wb)
            out[f"mask{i}"] = am.numpy()
        gen_golden_gqa._save("attn_weights_kvcache.npz", out)


if __name__ == "__main__":
    main()

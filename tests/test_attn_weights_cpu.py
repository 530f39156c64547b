"""The attention-weight oracle (oracle/attn_weights_oracle.py) against the reference's own `output_attentions=True` outputs
(tests/golden/attn_weights_*.npz, oracle/gen_golden_attn_weights.py): 1e-5 in fp32 and bit for bit in bf16, every row included — the
right-padded query rows and the uniform rows of queries with no visible key.  And the shipped cubin's attn_probs_kernel: HGMMA, no
local memory."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import attn_weights_oracle as W
from oracle import decoder_oracle as O
from oracle import gen_golden_attn_weights as GA
from oracle import gqa_oracle as G

GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")
BF = torch.bfloat16


def _from_bits(a):
    return torch.from_numpy(a.astype(np.int16)).view(BF)


def _oracle_layer(name, dtype):
    hidden, inter, heads, kv_heads, _, lens = GA.CASES[name]
    p, x, am, pos = GA.layer_case(name)
    pp = {k: v.to(dtype) for k, v in p.items()}
    cos, sin = O.rope_tables(hidden // heads, 2048, dtype=dtype)
    return W.layer_weights(x.to(dtype), pp, heads, kv_heads, cos, sin, pos, O.causal_additive_mask(len(lens), lens[0], dtype, am)), am


@pytest.mark.parametrize("name", sorted(GA.CASES))
def test_layer_weights_match_reference(name):
    g = np.load(os.path.join(GOLDEN_DIR, f"attn_weights_{name}.npz"))
    w32, am = _oracle_layer(name, torch.float32)
    assert np.array_equal(am.numpy(), g["mask"])
    torch.testing.assert_close(w32, torch.from_numpy(g["w"]), rtol=1e-5, atol=1e-5)
    wb, _ = _oracle_layer(name, BF)
    assert torch.equal(wb, _from_bits(g["w_bf16"]))


def test_row_semantics_of_padded_and_empty_samples():
    """g4d64: sample 1 has 45 of 72 tokens, sample 2 none.  Right-padded query rows are a softmax over the valid keys (not zero), rows
    with no visible key are uniform 1/kv_len in every column, masked keys are exactly 0."""
    g = np.load(os.path.join(GOLDEN_DIR, "attn_weights_g4d64.npz"))
    w, wb = torch.from_numpy(g["w"]), _from_bits(g["w_bf16"])
    S = w.shape[-1]
    pad_rows = w[1, :, 45:]
    assert float(pad_rows[..., 45:].abs().max()) == 0.0
    torch.testing.assert_close(pad_rows.sum(-1), torch.ones(pad_rows.shape[:-1]), rtol=1e-5, atol=1e-5)
    assert bool((pad_rows[..., :45] > 0).all())
    assert torch.equal(w[2], torch.full_like(w[2], 1.0 / S))
    assert torch.equal(wb[2], torch.full_like(wb[2], 1.0 / S).to(BF))
    causal_zero = torch.ones(S, S, dtype=torch.bool).triu(1)
    assert float(w[0][:, causal_zero].abs().max()) == 0.0


def test_kvcache_weights_match_reference():
    g = np.load(os.path.join(GOLDEN_DIR, "attn_weights_kvcache.npz"))
    hidden, inter, heads, kv_heads = [int(v) for v in g["shape"]]
    p, calls = G.cached_decode_scenario(hidden, inter, heads, kv_heads)
    w32 = W.run_cached_scenario(p, calls, heads, kv_heads)
    wb = W.run_cached_scenario(p, calls, heads, kv_heads, BF)
    assert len(calls) == 4
    for i, (x, am, _) in enumerate(calls):
        assert np.array_equal(am.numpy(), g[f"mask{i}"])
        assert w32[i].shape == (2, heads, x.shape[1], am.shape[1])
        torch.testing.assert_close(w32[i], torch.from_numpy(g[f"w{i}"]), rtol=1e-5, atol=1e-5)
        assert torch.equal(wb[i], _from_bits(g[f"w{i}_bf16"]))
    # the prefill's left-padded prompt positions of the shorter sample see no key: uniform over the whole row
    npad = int((calls[0][1][0] == 0).sum())
    assert npad > 0 and torch.equal(w32[0][0, :, :npad], torch.full_like(w32[0][0, :, :npad], 1.0 / calls[0][1].shape[1]))


def test_kernel_weights_restate_the_layer_path():
    """`kernel_weights` (token-major q / k, the kernel tests' yardstick) builds the same masks as the layer path."""
    name = "g4d64"
    hidden, inter, heads, kv_heads, _, lens = GA.CASES[name]
    p, x, am, pos = GA.layer_case(name)
    cos, sin = O.rope_tables(hidden // heads, 2048)
    q, k = W.qk_states(x, p, heads, kv_heads, cos, sin, pos)
    w = W.kernel_weights(q.transpose(1, 2), k.transpose(1, 2), seqlens=torch.tensor(lens))
    assert torch.equal(w, _oracle_layer(name, torch.float32)[0])


def test_attn_probs_kernel_is_hgmma_without_local_memory():
    from dreamllm_b200 import _lib
    _lib.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    bodies = [f for f in re.split(r"Function : ", sass)[1:] if "attn_probs_kernel" in f.split("\n", 1)[0]]
    assert len(bodies) == 4                                          # d 64 / 128 x causal / not
    for body in bodies:
        assert "HGMMA" in body and "UTMALDG" in body
        assert not re.search(r"\b(LDL|STL)\b", body), "local-memory access (spill)"
    res = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    usage = re.findall(r"Function (\S*attn_probs_kernel\S*):\s*\n\s*(.*)", res)
    assert len(usage) == 4, res[:2000]
    for fn, line in usage:
        assert re.search(r"\bLOCAL:0\b", line) and re.search(r"\bSTACK:0\b", line), (fn, line)

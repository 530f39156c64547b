"""Attention weights (`output_attentions=True`) on the GPU: `ops.attn_probs` (attn_probs_kernel) against the eager oracle
(oracle/attn_weights_oracle.py) under the like-for-like rule of DESIGN §2, and the decoder layer / model against the reference's own
weights (tests/golden/attn_weights_*.npz), with hidden states and gradients bit-identical to `output_attentions=False`."""
import os

import numpy as np
import pytest
import torch

from oracle import attn_weights_oracle as W
from oracle import gen_golden_attn_weights as GA
from oracle import gqa_oracle as G

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")


def _visible(B, Sq, Skv, causal=True, seqlens=None, kv_mask=None):
    """[B, 1, Sq, Skv] bool: the keys a query row may attend to (the reference's 4-D mask is 0 there)."""
    vis = torch.ones(B, 1, Sq, Skv, dtype=torch.bool)
    if causal:
        vis &= (torch.arange(Skv)[None] <= torch.arange(Sq)[:, None] + (Skv - Sq))[None, None]
    if seqlens is not None:
        vis &= (torch.arange(Skv)[None] < torch.as_tensor(seqlens)[:, None])[:, None, None, :]
    if kv_mask is not None:
        vis &= kv_mask.bool()[:, None, None, :Skv]
    return vis


def _check(ours, ref32, refbf, vis):
    """Like-for-like: err(ours, ref fp32) <= 1.5 err(ref bf16, ref fp32) on the rows with a visible key; rows without one bit-exact
    (uniform 1/Skv); masked keys of the other rows exactly 0."""
    ours = ours.cpu()
    assert not torch.isnan(ours.float()).any(), "element left unwritten"
    nh = ours.shape[1]
    vis = vis.expand(-1, nh, -1, -1)
    uni = ~vis.any(-1)
    assert torch.equal(ours[uni], refbf[uni])
    assert torch.equal(ours[uni], torch.full_like(ours[uni], 1.0 / ours.shape[-1]).to(BF))
    rows = ~uni
    masked = ~vis & rows[..., None]
    assert float(ours.float()[masked].abs().max() if masked.any() else 0.0) == 0.0
    if rows.any():
        o, r, rb = ours.float()[rows], ref32[rows], refbf.float()[rows]
        e_o, e_r = float((o - r).abs().mean()), float((rb - r).abs().mean())
        assert e_o <= 1.5 * e_r + 1e-6, f"ours {e_o:.3e} vs reference-bf16 {e_r:.3e}"
        assert float((o - r).abs().max()) <= 2 * float((rb - r).abs().max()) + 4e-3


def _nan_out(B, nh, Sq, Skv):
    return torch.full((B, nh, Sq, Skv), float("nan"), dtype=BF, device="cuda")


@pytest.mark.parametrize("S", [1, 63, 200, 257])
@pytest.mark.parametrize("nh,nkv", [(8, 8), (8, 2), (4, 1)])
@pytest.mark.parametrize("d", [64, 128])
def test_attn_probs_vs_oracle(d, nh, nkv, S):
    """Causal self-attention over a fused q|k|v buffer with right padding: a full sample, an empty one and a length that is not a multiple
    of 64 (right-padded query rows are a softmax over the valid keys; the empty sample's rows are uniform)."""
    from dreamllm_b200 import ops
    B = 3
    lens = [S, 0, max(1, (S * 2) // 3 | 1)]
    g = torch.Generator().manual_seed(100 * d + 10 * nkv + S)
    buf = torch.randn(B, S, nh + 2 * nkv, d, generator=g).to(BF)
    q, k = buf[:, :, :nh], buf[:, :, nh:nh + nkv]
    bd = buf.cuda()                                      # head slices of one buffer: the token stride stays (nh + 2 nkv) d at S == 1
    qd, kd, vd = bd[:, :, :nh], bd[:, :, nh:nh + nkv], bd[:, :, nh + nkv:]
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    _, lse = ops.attn_fwd(qd, kd, vd, causal=True, seqlens=sl)
    out = ops.attn_probs(qd, kd, lse, causal=True, seqlens=sl, out=_nan_out(B, nh, S, S))
    torch.cuda.synchronize()
    ref32 = W.kernel_weights(q.float(), k.float(), seqlens=lens)
    refbf = W.kernel_weights(q, k, seqlens=lens, dtype=BF)
    _check(out, ref32, refbf, _visible(B, S, S, seqlens=lens))


@pytest.mark.parametrize("Sq,Skv", [(1, 201), (5, 88), (88, 88), (3, 130)])
@pytest.mark.parametrize("d", [64, 128])
def test_attn_probs_kvcache_vs_oracle(d, Sq, Skv):
    """kv-cache reads: keys are the first Skv of 256 cache rows, bottom-right causal mask, a left-padded sample (key mask), odd Skv (rows
    not 16-byte aligned), single-token decode.  With Sq == Skv the left-padded prompt positions see no key: uniform rows."""
    from dreamllm_b200 import ops
    B, nh, nkv, max_len = 2, 8, 2, 256
    g = torch.Generator().manual_seed(7 * d + Sq + Skv)
    kc = torch.zeros(B, max_len, nkv, d, dtype=BF)
    vc = torch.zeros(B, max_len, nkv, d, dtype=BF)
    kc[:, :Skv] = torch.randn(B, Skv, nkv, d, generator=g).to(BF)
    vc[:, :Skv] = torch.randn(B, Skv, nkv, d, generator=g).to(BF)
    q = torch.randn(B, Sq, nh, d, generator=g).to(BF)
    mask = torch.ones(B, max_len, dtype=torch.uint8)
    mask[1, :30] = 0
    qd, kcd, vcd, md = q.cuda(), kc.cuda(), vc.cuda(), mask.cuda()
    _, lse = ops.attn_fwd_cache(qd, kcd, vcd, Skv, causal=True, kv_mask=md, return_lse=True)
    out = ops.attn_probs(qd, kcd, lse, causal=True, kv_len=Skv, kv_mask=md, out=_nan_out(B, nh, Sq, Skv))
    torch.cuda.synchronize()
    ref32 = W.kernel_weights(q.float(), kc[:, :Skv].float(), kv_mask=mask[:, :Skv])
    refbf = W.kernel_weights(q, kc[:, :Skv], kv_mask=mask[:, :Skv], dtype=BF)
    _check(out, ref32, refbf, _visible(B, Sq, Skv, kv_mask=mask))
    assert torch.equal(ops.attn_fwd_cache(qd, kcd, vcd, Skv, causal=True, kv_mask=md), ops.attn_fwd_cache(qd, kcd, vcd, Skv, kv_mask=md,
                                                                                                       return_lse=True)[0])


def test_attn_probs_rejects_what_the_forward_rejects():
    from dreamllm_b200._lib import lib
    L = lib()
    q = torch.zeros(1, 64, 6, 64, dtype=BF, device="cuda")
    lse = torch.zeros(1, 6, 64, dtype=torch.float32, device="cuda")
    probs = torch.empty(1, 6, 64, 64, dtype=BF, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    args = lambda nkv, d, S, Skv, p=probs.data_ptr(): (q.data_ptr(), q.data_ptr(), lse.data_ptr(), p, None, None, 0, 1, S, Skv, Skv, 6,  # noqa: E731
                                                       nkv, d, 6 * 64, 6 * 64, 1, 0.125, st)
    err = lambda rc: L.dllm_error_string(rc).decode()                                                                           # noqa: E731
    for nkv in (4, 0):
        assert err(L.dllm_attn_probs_gqa(*args(nkv, 64, 64, 64))) == "invalid shape / size"
    assert err(L.dllm_attn_probs_gqa(*args(6, 64, 64, 32))) == "invalid shape / size"                  # causal with Skv < S
    assert err(L.dllm_attn_probs_gqa(*args(6, 96, 64, 64))) == err(-6)                                  # head dim
    assert err(L.dllm_attn_probs_gqa(*args(6, 64, 64, 64, probs.data_ptr() + 2))) == err(-2)           # misaligned output


# ------------------------------------------------------------------------------------------------ decoder layer / model
def _layer(hidden, inter, heads, kv_heads, p):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer
    cfg = DreamLLMConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=heads, num_key_value_heads=kv_heads,
                         num_hidden_layers=1)
    layer = DreamLLMDecoderLayer(cfg)
    sd = {k: v.clone() for k, v in p.items()}
    sd["self_attn.rotary_emb.inv_freq"] = layer.self_attn.rotary_emb.inv_freq.clone()
    layer.load_state_dict(sd)
    return layer.to(device="cuda", dtype=BF)


def _bf(a):
    return torch.from_numpy(a.astype(np.int16)).view(BF)


@pytest.mark.parametrize("name", sorted(GA.CASES))
def test_layer_weights_vs_reference_golden(name):
    """The layer's weights against the reference layer's own: fp32 run as the yardstick, its bf16 run as the error budget."""
    hidden, inter, heads, kv_heads, _, lens = GA.CASES[name]
    g = np.load(os.path.join(GOLDEN_DIR, f"attn_weights_{name}.npz"))
    p, x, am, _ = GA.layer_case(name)
    layer = _layer(hidden, inter, heads, kv_heads, p)
    y, w = layer(x.to(BF).cuda(), attention_mask=am.cuda(), output_attentions=True)
    torch.cuda.synchronize()
    assert w.shape == (len(lens), heads, lens[0], lens[0]) and w.dtype == BF and w.is_contiguous()
    _check(w, torch.from_numpy(g["w"]), _bf(g["w_bf16"]), _visible(len(lens), lens[0], lens[0], seqlens=list(lens)))


def test_layer_outputs_and_gradients_bit_identical_with_weights_on():
    from dreamllm_b200 import ops
    hidden, inter, heads, kv_heads, _, lens = GA.CASES["g4d64"]
    p, x, am, _ = GA.layer_case("g4d64")
    layer = _layer(hidden, inter, heads, kv_heads, p)
    gy = torch.randn(x.shape, generator=torch.Generator().manual_seed(3)).to(BF).cuda()
    runs = []
    for oa in (False, True):
        layer.zero_grad(set_to_none=True)
        xc = x.to(BF).cuda().requires_grad_(True)
        n0 = ops.LAUNCHES.count
        outs = layer(xc, attention_mask=am.cuda(), output_attentions=oa)
        assert len(outs) == (2 if oa else 1)
        if oa:
            assert not outs[1].requires_grad and outs[1].grad_fn is None
        outs[0].backward(gy)
        runs.append((outs[0].detach(), xc.grad, {k: q.grad.clone() for k, q in layer.named_parameters()}, ops.LAUNCHES.count - n0))
    (y0, dx0, g0, n0), (y1, dx1, g1, n1) = runs
    assert torch.equal(y0, y1) and torch.equal(dx0, dx1)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    assert n1 == n0 + 1                                                         # the one attn_probs launch


def test_cached_layer_weights_vs_reference_golden():
    """Left-padded prefill + 3 decode steps through the kv-cache: [B, nh, S_new, past + S_new] per call, the prompt's pad positions
    uniform, against the reference's `past_key_value` run."""
    from dreamllm_b200.modeling_dreamllm import KVCache
    g = np.load(os.path.join(GOLDEN_DIR, "attn_weights_kvcache.npz"))
    hidden, inter, heads, kv_heads = [int(v) for v in g["shape"]]
    p, calls = G.cached_decode_scenario(hidden, inter, heads, kv_heads)
    layer = _layer(hidden, inter, heads, kv_heads, p).eval()
    cache = KVCache(1, 2, 128, kv_heads, hidden // heads, "cuda")
    for i, (x, am, pos) in enumerate(calls):
        cache.set_mask(am.cuda())
        with torch.no_grad():
            y, w, (c, li) = layer(x.cuda().to(BF), position_ids=pos.cuda(), past_key_value=(cache, 0), use_cache=True,
                                  output_attentions=True)
        past = cache.len
        cache.len += x.shape[1]
        assert c is cache and li == 0
        assert w.shape == (2, heads, x.shape[1], past + x.shape[1])
        _check(w, torch.from_numpy(g[f"w{i}"]), _bf(g[f"w{i}_bf16"]), _visible(2, x.shape[1], past + x.shape[1], kv_mask=am))


def _lm(layers=2, kv_heads=2, **kw):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=512, hidden_size=512, intermediate_size=1024, num_hidden_layers=layers, num_attention_heads=8,
                         num_key_value_heads=kv_heads, max_position_embeddings=512, **kw)
    return DreamLLMForCausalMLM(cfg).to(device="cuda", dtype=BF)


def _batch(B=2, S=96, pad=30):
    ids = torch.randint(1, 512, (B, S), generator=torch.Generator().manual_seed(5)).cuda()
    am = torch.ones_like(ids)
    am[1, S - pad:] = 0
    return ids, am, ids.masked_fill(am == 0, -100)


def test_causal_lm_attentions_text_batch():
    m = _lm(layers=3)
    ids, am, labels = _batch()
    out = m(input_ids=ids, attention_mask=am, labels=labels, output_attentions=True)
    assert len(out.attentions) == 3
    for w in out.attentions:
        assert w.shape == (2, 8, 96, 96) and w.dtype == BF and not w.requires_grad
    ref = m(input_ids=ids, attention_mask=am, labels=labels)
    assert ref.attentions is None and torch.equal(out.loss, ref.loss)
    # the layer's own weights, from the model's hidden states
    hs = m(input_ids=ids, attention_mask=am, output_hidden_states=True, output_attentions=True)
    for li, layer in enumerate(m.model.layers):
        assert torch.equal(layer(hs.hidden_states[li], attention_mask=am, output_attentions=True)[1], hs.attentions[li])


def test_causal_lm_attentions_image_spliced_batch():
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    from dreamllm_b200.modeling_plugins import CLIPVisionEmbedding, DreamEmbedding
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=32008, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2)
    m = DreamLLMForCausalMLM(cfg)
    clip = CLIPVisionEmbedding(dict(hidden_size=256, intermediate_size=512, num_hidden_layers=3, num_attention_heads=4, image_size=56,
                                    patch_size=14), embed_hidden_size=256)
    m.model.attach_plugins(clip, DreamEmbedding(num_dream_queries=8, embed_hidden_size=256), image_start_id=32003, dream_start_id=32006)
    m = m.to(device="cuda", dtype=BF)
    P = clip.embed_len
    ids = torch.full((2, 64), 32000)
    ids[0, :P + 6] = torch.tensor([1, 32003] + [32002] * P + [32004, 5, 6, 2])
    ids[1, :P + 5] = torch.tensor([1, 32003] + [32002] * P + [32004, 7, 2])
    labels = ids.masked_fill(ids >= 32000, -100)
    am = (ids != 32000).long()
    imgs = torch.randn(2, 3, 56, 56).to(BF).cuda()
    out = m(input_ids=ids.cuda(), images=imgs, attention_mask=am.cuda(), labels=labels.cuda(), input_ids_cpu=ids, output_attentions=True)
    assert len(out.attentions) == 2 and all(w.shape == (2, 2, 64, 64) for w in out.attentions)
    ref = m(input_ids=ids.cuda(), images=imgs, attention_mask=am.cuda(), labels=labels.cuda(), input_ids_cpu=ids)
    assert torch.equal(out.loss, ref.loss)
    # sample 1: 22 valid tokens; its right-padded query rows attend to those keys only and sum to 1
    w = out.attentions[0][1].float()
    n = int(am[1].sum())
    assert float(w[:, n:, n:].abs().max()) == 0.0
    torch.testing.assert_close(w[:, n:, :n].sum(-1), torch.ones(2, 64 - n, device="cuda"), rtol=2e-2, atol=2e-2)


def test_config_flags_and_additional_log_info():
    import logging
    m = _lm(layers=3)
    ids, am, labels = _batch()
    m.config.output_attentions = True
    out = m(input_ids=ids, attention_mask=am, labels=labels)
    assert len(out.attentions) == 3 and set(out.additional_log_info) == {"lm_loss", "vm_loss"}
    m.config.output_attentions = False
    assert m(input_ids=ids, attention_mask=am, labels=labels).attentions is None
    m.config.log_attentions = True                       # forces the weights on and logs their max |.|
    m.config.log_hidden_states = True
    out = m(input_ids=ids, attention_mask=am, labels=labels, output_attentions=False, output_hidden_states=True)
    info = out.additional_log_info
    keys = [k for k in info if k not in ("lm_loss", "vm_loss")]
    assert keys == ["hidden_states_layer-1", "attentions_layer0", "hidden_states_layer0", "attentions_layer1", "hidden_states_layer1",
                    "attentions_layer2", "hidden_states_layer2"]                  # the reference's insertion order (:988-1032)
    for i in range(3):
        assert isinstance(info[f"attentions_layer{i}"], float)
        assert info[f"attentions_layer{i}"] == float(out.attentions[i].abs().max())
        assert info[f"hidden_states_layer{i - 1}"] == float(out.hidden_states[i].abs().max())
    assert info["hidden_states_layer2"] == float(out.hidden_states[3].abs().max())      # the final normed output
    m.config._flash_attn_2_enabled = True                # the reference switches the weights off under flash-attn 2, with a warning
    from dreamllm_b200 import modeling_dreamllm as MD
    MD._warn_once.cache_clear()
    seen = []
    handler = logging.Handler()
    handler.emit = lambda r: seen.append(r.getMessage())
    MD.logger.addHandler(handler)
    try:
        out = m(input_ids=ids, attention_mask=am, labels=labels, output_attentions=True)
    finally:
        MD.logger.removeHandler(handler)
    assert out.attentions is None and not any(k.startswith("attentions_") for k in out.additional_log_info)
    assert any("output_attentions" in s for s in seen)


def test_cached_model_decode_returns_weights():
    m = _lm().eval()
    ids = torch.randint(1, 512, (2, 40), generator=torch.Generator().manual_seed(9)).cuda()
    am = torch.ones_like(ids)
    am[0, :7] = 0                                        # left-padded prompt
    with torch.no_grad():
        out = m(input_ids=ids, attention_mask=am, use_cache=True, output_attentions=True)
        assert [tuple(w.shape) for w in out.attentions] == [(2, 8, 40, 40)] * 2
        assert torch.equal(out.attentions[0][0, :, :7].float(), torch.full((8, 7, 40), 1 / 40, device="cuda").to(BF).float())
        am2 = torch.cat([am, torch.ones(2, 1, dtype=am.dtype, device="cuda")], 1)
        step = m(input_ids=ids[:, -1:], attention_mask=am2, past_key_values=out.past_key_values, use_cache=True, output_attentions=True)
    assert [tuple(w.shape) for w in step.attentions] == [(2, 8, 1, 41)] * 2
    assert float(step.attentions[0][0, :, :, :7].float().abs().max()) == 0.0


def _count_probs(monkeypatch):
    from dreamllm_b200 import ops
    n = [0]
    real = ops.attn_probs

    def spy(*a, **k):
        n[0] += 1
        return real(*a, **k)
    monkeypatch.setattr(ops, "attn_probs", spy)
    return n


def test_checkpointing_materialises_weights_once_per_layer(monkeypatch):
    n = _count_probs(monkeypatch)

    def run(oa):
        m = _lm(layers=3).train()
        m.gradient_checkpointing_enable()
        ids, am, labels = _batch()
        out = m(input_ids=ids, attention_mask=am, labels=labels, output_attentions=oa)
        out.loss.backward()
        return out, {k: p.grad.clone() for k, p in m.named_parameters()}
    o0, g0 = run(False)
    assert n[0] == 0
    o1, g1 = run(True)
    assert n[0] == 3                                     # forward only: the recompute inside backward reuses the weights
    assert torch.equal(o0.loss, o1.loss) and len(o1.attentions) == 3
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


def test_weights_kernel_never_runs_when_off(monkeypatch):
    n = _count_probs(monkeypatch)
    m = _lm()
    ids, am, labels = _batch()
    m(input_ids=ids, attention_mask=am, labels=labels).loss.backward()
    with torch.no_grad():
        m.eval()
        m.generate(ids[:, :20], max_new_tokens=3)
    assert n[0] == 0

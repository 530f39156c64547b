"""Packed (unpadded) batches on the GPU: the variable-length attention kernels, the packed decoder layer and the packed causal LM.

A packed batch is the right-padded batch with its pad rows deleted, and the kernels align their tiles to the start of every sample
exactly as the padded layout does.  So the yardsticks are the existing ones: each sample of a packed attention call must equal, bit for
bit, `dllm_attn_fwd_gqa` / `dllm_attn_bwd_gqa` run on that sample alone; against the reference's eager math the criterion is
test_attn_gpu.py's; layer and model are held to the CPU oracle run sample by sample and to this package's own padded path."""
import math

import pytest
import torch

from oracle import decoder_oracle as O
from oracle import gqa_oracle as G

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
SENTINEL = 777.0          # finite, exactly representable in bf16 / fp32: a row still holding it was never written


def _cu(lens):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32)


def _views(buf, nh, nkv, d):
    """q [.., nh, d], k and v [.., nkv, d]: head-slice views of a fused [.., nh + 2 nkv, d] projection buffer"""
    return buf[..., :nh, :], buf[..., nh:nh + nkv, :], buf[..., nh + nkv:, :]


def _packed_fwd_bwd(buf, dout, cu, max_len, nh, nkv, d, causal):
    from dreamllm_b200 import ops
    out, lse = ops.attn_fwd_varlen(*_views(buf, nh, nkv, d), cu, max_len, causal=causal)
    dbuf = torch.full_like(buf, SENTINEL)
    ops.attn_bwd_varlen(dout, *_views(buf, nh, nkv, d), out, lse, *_views(dbuf, nh, nkv, d), cu, max_len, causal=causal)
    return out, lse, dbuf


KERNEL_CASES = [
    # lens, nh, nkv, d, causal                                                   T = 777 below: not a multiple of 8
    ([1, 63, 64, 65, 127, 128, 129, 200], 2, 2, 128, True),
    ([1, 63, 64, 65, 127, 128, 129, 200], 4, 2, 64, False),
    ([200, 129, 128, 127, 65, 64, 63, 1], 4, 2, 64, True),
    ([0, 200, 0, 129, 65, 0], 4, 1, 128, True),                  # MQA; empty samples first, in the middle and last
    ([0, 77, 0, 0, 130, 0], 2, 2, 64, False),
    ([2100, 300, 5], 2, 1, 128, True),                           # a sample above 2048
    ([333], 2, 2, 64, True),                                     # B = 1
    ([129, 0, 64, 5], 4, 2, 128, False),
]


@pytest.mark.parametrize("lens,nh,nkv,d,causal", KERNEL_CASES)
def test_each_sample_equals_the_padded_kernels_on_that_sample_alone_bit_for_bit(lens, nh, nkv, d, causal):
    from dreamllm_b200 import ops
    T = sum(lens)
    g = torch.Generator().manual_seed(1000 + T + nkv)
    buf = torch.randn(T, nh + 2 * nkv, d, generator=g).to(BF).cuda()          # q | k | v slices of one fused buffer
    dout = (torch.randn(T, nh * d, generator=g) * 0.5).to(BF).cuda()
    cu = _cu(lens)
    cud = cu.cuda()
    out, lse, dbuf = _packed_fwd_bwd(buf, dout, cud, max(lens), nh, nkv, d, causal)
    out2, lse2, dbuf2 = _packed_fwd_bwd(buf, dout, cud, max(lens), nh, nkv, d, causal)
    torch.cuda.synchronize()
    assert torch.equal(out, out2) and torch.equal(lse, lse2) and torch.equal(dbuf, dbuf2)      # deterministic backward
    assert not bool((dbuf == SENTINEL).any())                                                    # every gradient row was written
    assert bool(torch.isfinite(out.float()).all()) and bool(torch.isfinite(lse).all())
    for b, n in enumerate(lens):
        if n == 0:
            continue
        s, e = int(cu[b]), int(cu[b + 1])
        one = buf[s:e].clone()[None]                                             # [1, n, nh + 2 nkv, d]: the sample on its own
        q, k, v = _views(one, nh, nkv, d)
        o1, l1 = ops.attn_fwd(q, k, v, causal=causal)
        d1 = torch.full_like(one, SENTINEL)
        ops.attn_bwd(dout[s:e].clone()[None], q, k, v, o1, l1, *_views(d1, nh, nkv, d), causal=causal)
        assert torch.equal(out[s:e], o1[0]), f"out of sample {b} (len {n})"
        assert torch.equal(lse[:, s:e], l1[0]), f"lse of sample {b} (len {n})"
        for name, got, want in zip(("dq", "dk", "dv"), _views(dbuf[s:e], nh, nkv, d), _views(d1[0], nh, nkv, d)):
            assert torch.equal(got, want), f"{name} of sample {b} (len {n})"


def test_larger_grid_than_needed_and_buffers_next_to_the_outputs_are_left_alone():
    """`max_seqlen` only has to bound the lengths, and nothing outside the T rows is written: out / lse / dqkv are carved out of larger
    sentinel-filled allocations here."""
    from dreamllm_b200 import ops
    lens, nh, nkv, d = [70, 130, 3], 2, 1, 64
    T = sum(lens)
    g = torch.Generator().manual_seed(5)
    buf = torch.randn(T, nh + 2 * nkv, d, generator=g).to(BF).cuda()
    dout = torch.randn(T, nh * d, generator=g).to(BF).cuda()
    cu = _cu(lens).cuda()
    a = _packed_fwd_bwd(buf, dout, cu, 130, nh, nkv, d, True)
    b = _packed_fwd_bwd(buf, dout, cu, T, nh, nkv, d, True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    big = torch.full((T + 256, nh + 2 * nkv, d), SENTINEL, dtype=BF, device="cuda")
    dq, dk, dv = _views(big[128:128 + T], nh, nkv, d)
    ops.attn_bwd_varlen(dout, *_views(buf, nh, nkv, d), a[0], a[1], dq, dk, dv, cu, 130, causal=True)
    torch.cuda.synchronize()
    assert torch.equal(big[128:128 + T], a[2]) and bool((big[:128] == SENTINEL).all()) and bool((big[128 + T:] == SENTINEL).all())


def _ref_core(q, k, v, causal):
    """q [1,S,nh,d], k/v [1,S,nkv,d] -> out [1,S,nh*d]: the reference's eager math (modeling_dreamllm.py:357-379) in the input dtype
    after `repeat_kv`, additive finfo.min mask, fp32 softmax cast back to the input dtype.  In bf16 it is the reference's own bf16 path."""
    B, S, nh, d = q.shape
    dt = q.dtype
    qh = q.transpose(1, 2)
    kh, vh = (G.repeat_kv(t.transpose(1, 2), nh // k.shape[2]) for t in (k, v))
    w = torch.matmul(qh, kh.transpose(2, 3)) / math.sqrt(d)
    mask = torch.zeros(B, 1, S, S, dtype=dt)
    if causal:
        mask = mask.masked_fill(torch.ones(S, S, dtype=torch.bool).triu(1), torch.finfo(dt).min)
    w = torch.max(w + mask, torch.tensor(torch.finfo(dt).min, dtype=dt))
    p = torch.softmax(w, dim=-1, dtype=torch.float32).to(dt)
    return torch.matmul(p, vh).transpose(1, 2).reshape(B, S, nh * d)


@pytest.mark.parametrize("lens,nh,nkv,d,causal", [([200, 77, 129, 1], 2, 2, 128, True), ([150, 64, 0, 33], 4, 2, 64, False),
                                                  ([300, 65], 4, 1, 128, True)])
def test_packed_kernels_vs_eager_reference_per_sample(lens, nh, nkv, d, causal):
    T = sum(lens)
    g = torch.Generator().manual_seed(300 + T)
    buf = torch.randn(T, nh + 2 * nkv, d, generator=g).to(BF)
    dout = (torch.randn(T, nh * d, generator=g) * 0.5).to(BF)
    cu = _cu(lens)
    out, _, dbuf = _packed_fwd_bwd(buf.cuda(), dout.cuda(), cu.cuda(), max(lens), nh, nkv, d, causal)
    torch.cuda.synchronize()
    ours = dict(zip(("dq", "dk", "dv"), (t.cpu().float() for t in _views(dbuf, nh, nkv, d))))
    ours["out"] = out.cpu().float()
    ref32 = {k: torch.zeros_like(v) for k, v in ours.items()}
    refbf = {k: torch.zeros_like(v) for k, v in ours.items()}
    for b, n in enumerate(lens):
        if n == 0:
            continue
        s, e = int(cu[b]), int(cu[b + 1])
        for dt, dst in ((torch.float32, ref32), (BF, refbf)):
            q, k, v = (t[None].to(dt).clone().requires_grad_(True) for t in _views(buf[s:e], nh, nkv, d))
            o = _ref_core(q, k, v, causal)
            o.backward(dout[s:e][None].to(dt))
            dst["out"][s:e] = o.detach()[0].float()
            for name, t in (("dq", q), ("dk", k), ("dv", v)):
                dst[name][s:e] = t.grad[0].float()
    torch.testing.assert_close(ours["out"], ref32["out"], rtol=2e-2, atol=2e-2)
    for name in ("out", "dq", "dk", "dv"):
        err = (ours[name] - ref32[name]).abs()
        scale = float(ref32[name].abs().max())
        assert float(err.max()) < 3e-2 * scale + 1e-3, f"{name}: max err {float(err.max())} vs scale {scale}"
        e_r = float((refbf[name] - ref32[name]).abs().mean())
        assert float(err.mean()) <= 1.5 * e_r + 1e-5 * scale, f"{name}: ours {float(err.mean()):.3e} vs reference-bf16 {e_r:.3e}"


def test_bad_arguments_are_reported_by_the_c_abi():
    from dreamllm_b200._lib import lib
    L = lib()
    T, nh, nkv, d = 64, 2, 2, 64
    buf = torch.zeros(T, nh + 2 * nkv, d, dtype=BF, device="cuda")
    q, k, v = _views(buf, nh, nkv, d)
    out = torch.empty(T, nh * d, dtype=BF, device="cuda")
    lse = torch.empty(nh, T, dtype=torch.float32, device="cuda")
    cu = _cu([T]).cuda()
    ld, st = buf.stride(0), torch.cuda.current_stream().cuda_stream

    def fwd(cu_ptr=cu.data_ptr(), max_len=T, nkv_=nkv, d_=d, ld_o=nh * d):
        return L.dllm_error_string(L.dllm_attn_fwd_varlen(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), cu_ptr,
                                                          1, T, max_len, nh, nkv_, d_, ld, ld, ld_o, 1, 0.125, st)).decode()
    ok, shape = L.dllm_error_string(0).decode(), L.dllm_error_string(-1).decode()
    assert fwd() == ok
    assert fwd(cu_ptr=None) == shape and fwd(max_len=0) == shape and fwd(max_len=T + 1) == shape and fwd(nkv_=3) == shape
    assert fwd(d_=96) == L.dllm_error_string(-6).decode() and fwd(ld_o=nh * d + 4) == L.dllm_error_string(-2).decode()
    ws = torch.empty(L.dllm_attn_bwd_varlen_workspace_bytes(T, nh, d), dtype=torch.uint8, device="cuda")
    args = [out.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), q.data_ptr(), k.data_ptr(),
            v.data_ptr(), None, ws.data_ptr(), ws.numel(), 1, T, T, nh, nkv, d, ld, ld, nh * d, ld, ld, 1, 0.125, st]
    assert L.dllm_error_string(L.dllm_attn_bwd_varlen(*args)).decode() == shape                  # NULL cu_seqlens
    args[9], args[11] = cu.data_ptr(), ws.numel() - 4
    assert L.dllm_error_string(L.dllm_attn_bwd_varlen(*args)).decode() == shape                  # workspace too small
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ decoder layer
def _err(a, ref):
    e = (a.float() - ref.float()).abs().flatten()
    k = max(1, int(e.numel() * 0.999))
    return float(e.mean()), float(e.kthvalue(k).values)


def _like_for_like(name, ours, refb, gold):
    """test_decoder_layer_gpu.py's criterion: as close to the fp32 oracle as the oracle's own bf16 run is"""
    m_o, p_o = _err(ours, gold)
    m_r, p_r = _err(refb, gold)
    scale = float(gold.abs().mean()) + 1e-12
    msg = f"{name}: ours mean {m_o:.3e} p99.9 {p_o:.3e} | oracle-bf16 mean {m_r:.3e} p99.9 {p_r:.3e} | |oracle| {scale:.3e}"
    assert m_o <= 1.25 * m_r + 2e-3 * scale, msg
    assert p_o <= 1.5 * p_r + 2e-2 * scale, msg


def _layer(hidden, inter, heads, kv_heads, p):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer
    cfg = DreamLLMConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=heads, num_key_value_heads=kv_heads,
                         num_hidden_layers=1)
    layer = DreamLLMDecoderLayer(cfg)
    sd = {k: v.clone() for k, v in p.items()}
    sd["self_attn.rotary_emb.inv_freq"] = layer.self_attn.rotary_emb.inv_freq.clone()
    layer.load_state_dict(sd)
    return layer.to(device="cuda", dtype=BF)


def _oracle_layer_per_sample(x, gy, lens, p, heads, kv_heads, dt):
    """fp32 / bf16 CPU oracle, one sample at a time: y, dx over the packed rows and the summed weight gradients"""
    hidden = x.shape[-1]
    pp = {k: v.to(dt).clone().requires_grad_(True) for k, v in p.items()}
    cos, sin = O.rope_tables(hidden // heads, 2048, dtype=dt)
    xs = x.to(dt).clone().requires_grad_(True)
    ys, s = [], 0
    for n in lens:
        if n:
            xi = xs[s:s + n][None]
            pos = torch.arange(n)[None]
            ys.append(G.decoder_layer(xi, pp, heads, kv_heads, cos, sin, pos, O.causal_additive_mask(1, n, dt, None))[0])
        s += n
    y = torch.cat(ys, 0)
    y.backward(gy.to(dt))
    return y.detach(), xs.grad, {k: v.grad for k, v in pp.items()}


@pytest.mark.parametrize("heads,kv_heads", [(4, 4), (8, 2)])
def test_packed_decoder_layer_vs_oracle_and_padded_path(heads, kv_heads):
    hidden, inter, lens = 512, 1024, [200, 77, 0, 129, 1]
    T, B, S = sum(lens), len(lens), max(lens)
    p = G.init_layer_params(hidden, inter, 11, heads, kv_heads)
    g = torch.Generator().manual_seed(12)
    x = torch.randn(T, hidden, generator=g).to(BF)
    gy = (torch.randn(T, hidden, generator=g) * 0.1).to(BF)
    y32, dx32, dw32 = _oracle_layer_per_sample(x.float(), gy.float(), lens, p, heads, kv_heads, torch.float32)
    ybf, dxbf, dwbf = _oracle_layer_per_sample(x, gy, lens, p, heads, kv_heads, BF)

    cu = _cu(lens)
    layer = _layer(hidden, inter, heads, kv_heads, p)
    xc = x.cuda()[None].requires_grad_(True)
    y = layer(xc, cu_seqlens=cu, max_seqlen=S)[0]                  # host cu_seqlens: validated and uploaded by the layer
    y.backward(gy.cuda()[None])
    torch.cuda.synchronize()
    assert y.shape == (1, T, hidden)
    _like_for_like("y", y[0].detach().cpu(), ybf, y32)
    _like_for_like("dx", xc.grad[0].cpu(), dxbf, dx32)
    named = dict(layer.named_parameters())
    for k in O.LAYER_KEYS:
        _like_for_like("d_" + k, named[k].grad.cpu(), dwbf[k], dw32[k])
    packed_grads = {k: named[k].grad.clone() for k in O.LAYER_KEYS}

    # this package's padded path on the same data: right-padded rows, dy zero on the pad rows
    valid = torch.arange(S)[None] < torch.tensor(lens)[:, None]
    xp, gp = torch.zeros(B, S, hidden, dtype=BF), torch.zeros(B, S, hidden, dtype=BF)
    xp[valid], gp[valid] = x, gy
    layer.zero_grad()
    xpc = xp.cuda().requires_grad_(True)
    yp = layer(xpc, attention_mask=valid.long().cuda())[0]
    yp.backward(gp.cuda())
    torch.cuda.synchronize()
    # the same kernels on the same rows in the same order, except the GEMMs' row tiling and the wgrad's K split: bf16 rounding
    torch.testing.assert_close(y[0].float().cpu(), yp.detach().cpu()[valid].float(), rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(xc.grad[0].float().cpu(), xpc.grad.cpu()[valid].float(), rtol=2e-2, atol=2e-3)
    for k in O.LAYER_KEYS:
        a, b = packed_grads[k].float(), named[k].grad.float()
        assert float((a - b).abs().mean()) <= 1e-2 * float(b.abs().mean()) + 1e-6, k


# ------------------------------------------------------------------------------------------------ causal LM
def _lm(kv_heads=2, layers=2, vocab=512, hidden=256):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=vocab, hidden_size=hidden, intermediate_size=2 * hidden, num_hidden_layers=layers,
                         num_attention_heads=4, num_key_value_heads=kv_heads, max_position_embeddings=512)
    return DreamLLMForCausalMLM(cfg)


def _text_batches(lens, vocab=512, seed=1):
    """The same ragged token lists as a right-padded batch and as a packed one (what the collator emits for either layout)."""
    from types import SimpleNamespace
    from dreamllm_b200.collator import DataCollatorForDreamLLMDataset
    g = torch.Generator().manual_seed(seed)
    ex = []
    for n in lens:
        ids = torch.randint(3, vocab, (n,), generator=g)
        lab = ids.clone()
        lab[: n // 3] = -100                                       # a prompt that carries no loss
        ex.append(dict(input_ids=ids, attention_mask=torch.ones(n, dtype=torch.long), labels=lab))
    tok = SimpleNamespace(pad_token_id=0)
    return DataCollatorForDreamLLMDataset(tok)(ex), DataCollatorForDreamLLMDataset(tok, pack=True)(ex)


MODEL_KEYS = ("input_ids", "attention_mask", "labels", "shifted_labels", "seqlens", "attention_mask_has_padding", "position_ids",
              "cu_seqlens", "max_seqlen")


def _step(m, batch, **extra):
    from dreamllm_b200.collator import to_device
    m.zero_grad()
    out = m(**{k: v for k, v in to_device(batch, "cuda").items() if k in MODEL_KEYS}, **extra)
    out.loss.backward()
    torch.cuda.synchronize()
    return out, {k: p.grad.detach().clone() for k, p in m.named_parameters()}


def test_packed_causal_lm_vs_oracle_and_padded_path():
    lens = [150, 40, 97, 1, 64]
    padded, packed = _text_batches(lens)
    m = _lm(kv_heads=4).to(device="cuda", dtype=BF).train()
    out_pk, g_pk = _step(m, packed)
    out_pd, g_pd = _step(m, padded)
    lpk, lpd = float(out_pk.loss.detach()), float(out_pd.loss.detach())
    assert abs(lpk - lpd) <= 2e-3 * abs(lpd)
    for k in g_pd:
        a, b = g_pk[k].float(), g_pd[k].float()
        assert float((a - b).abs().mean()) <= 2e-2 * float(b.abs().mean()) + 1e-7, k

    # CPU oracle, sample by sample: the masked-mean loss over all label tokens is the token-weighted mean of the per-sample losses
    sd = {k: v.detach().float().cpu() for k, v in m.state_dict().items()}
    results = {}
    for dt in (torch.float32, BF):
        w = {k: v.to(dt).clone().requires_grad_(True) for k, v in sd.items() if not k.endswith("inv_freq")}
        lay = [{k: w[f"model.layers.{i}.{k}"] for k in O.LAYER_KEYS} for i in range(2)]
        total, count = 0.0, 0
        for b, n in enumerate(lens):
            ids, lab = padded["input_ids"][b:b + 1, :n], padded["labels"][b:b + 1, :n]
            nlab = int((lab[:, 1:] != -100).sum())
            if nlab == 0:
                continue
            loss, _, _ = O.causal_lm(ids, lab, w["model.embed_tokens.weight"], lay, w["model.norm.weight"], w["lm_head.weight"], 4)
            total, count = total + loss.float() * nlab, count + nlab
        loss = total / count
        loss.backward()
        results[dt] = (float(loss.detach()), {k: v.grad for k, v in w.items()})
    l32, g32 = results[torch.float32]
    lbf, gbf = results[BF]
    assert count == packed["num_label_tokens"]
    assert abs(lpk - l32) <= 1.5 * abs(lbf - l32) + 2e-3 * abs(l32), (lpk, lbf, l32)
    for k in g32:
        _like_for_like("d_" + k, g_pk[k].cpu(), gbf[k], g32[k])


def test_packed_model_derives_positions_and_labels_like_the_collator():
    """Without the collator's `position_ids` / `shifted_labels` the model builds both on the device from `cu_seqlens`; same bits."""
    _, packed = _text_batches([33, 150, 7])
    m = _lm().to(device="cuda", dtype=BF).train()
    out_a, g_a = _step(m, packed)
    bare = {k: packed[k] for k in ("input_ids", "labels", "cu_seqlens", "max_seqlen")}
    out_b, g_b = _step(m, bare)
    assert torch.equal(out_a.loss, out_b.loss)
    for k in g_a:
        assert torch.equal(g_a[k], g_b[k]), k
    dev = dict(bare, cu_seqlens=packed["cu_seqlens"].cuda())       # boundaries already on the device: trusted, not read back
    assert torch.equal(_step(m, dev)[0].loss, out_a.loss)


def test_packed_gradient_checkpointing_is_bit_identical():
    _, packed = _text_batches([150, 40, 97, 64])
    m = _lm(layers=3).to(device="cuda", dtype=BF).train()
    out0, g0 = _step(m, packed)
    m.gradient_checkpointing_enable()
    out1, g1 = _step(m, packed)
    assert torch.equal(out0.loss, out1.loss)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


def test_packed_step_with_images_and_a_dream_query_diffusion_loss_matches_the_padded_step():
    from types import SimpleNamespace
    from dreamllm_b200.collator import DataCollatorForDreamLLMDataset, to_device
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    from dreamllm_b200.modeling_plugins import CLIPVisionEmbedding, DreamEmbedding, StableDiffusionHead
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=32008, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2)
    m = DreamLLMForCausalMLM(cfg)
    clip = CLIPVisionEmbedding(dict(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4, image_size=56,
                                    patch_size=14), embed_hidden_size=256)
    Q = 8
    dream = DreamEmbedding(num_dream_queries=Q, embed_hidden_size=256)
    m.stable_diffusion_head = StableDiffusionHead(dict(block_out_channels=(64, 128, 256, 256), attention_head_dim=(1, 2, 4, 4),
                                                       cross_attention_dim=128, vae=dict(block_out_channels=(64, 128, 128, 128))),
                                                  embed_hidden_size=256)
    m.model.attach_plugins(clip, dream, image_start_id=32003, dream_start_id=32006)
    m = m.to(device="cuda", dtype=BF).train()
    P = clip.embed_len
    g = torch.Generator().manual_seed(4)

    def sample(n_text, image, dreamq):
        ids = [1] + ([32003] + [32002] * P + [32004] if image else []) + torch.randint(5, 3000, (n_text,), generator=g).tolist()
        ids += ([32006] + [32002] * Q + [32007] if dreamq else []) + [2]
        ids = torch.tensor(ids)
        return dict(input_ids=ids, attention_mask=torch.ones_like(ids), labels=ids.masked_fill(ids >= 32000, -100),
                    images=torch.randn(1, 3, 56, 56, generator=g).to(BF) if image else None,
                    images_dm=(torch.rand(1, 3, 128, 128, generator=g) * 2 - 1).to(BF) if dreamq else None)
    ex = [sample(9, True, True), sample(30, False, False), sample(3, True, False), sample(14, False, True)]
    kw = dict(image_start_id=32003, dream_start_id=32006, clip_embed_len=P, dream_embed_len=Q)
    tok = SimpleNamespace(pad_token_id=32000)
    padded, packed = DataCollatorForDreamLLMDataset(tok, **kw)(ex), DataCollatorForDreamLLMDataset(tok, pack=True, **kw)(ex)
    draws = dict(vae_noise=torch.randn(2, 4, 16, 16, generator=g).cuda(), noise=torch.randn(2, 4, 16, 16, generator=g).cuda(),
                 timesteps=torch.tensor([17, 803]).cuda())
    keys = MODEL_KEYS + ("images", "images_dm", "input_ids_cpu", "splice_plan")
    res = []
    for batch in (packed, padded):
        m.zero_grad()
        out = m(**{k: v for k, v in to_device(batch, "cuda").items() if k in keys}, sd_kwargs=draws)
        out.loss.backward()
        torch.cuda.synchronize()
        res.append((out, {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}))
    (o_pk, g_pk), (o_pd, g_pd) = res
    for k in ("lm_loss", "vm_loss"):
        a, b = float(o_pk.additional_log_info[k]), float(o_pd.additional_log_info[k])
        assert b > 0 and abs(a - b) <= 1e-2 * b, (k, a, b)
    torch.testing.assert_close(o_pk.additional_log_info["dream_conditioning"].float(), o_pd.additional_log_info["dream_conditioning"].float(),
                               rtol=2e-2, atol=2e-2)
    assert set(g_pk) == set(g_pd) and "model.dream_embedding.dream_queries" in g_pk
    for k in g_pd:
        a, b = g_pk[k].float(), g_pd[k].float()
        assert float((a - b).abs().mean()) <= 5e-2 * float(b.abs().mean()) + 1e-7, k


def test_packed_input_error_paths():
    from dreamllm_b200.modeling_dreamllm import KVCache
    _, packed = _text_batches([20, 30])
    m = _lm().to(device="cuda", dtype=BF).eval()
    ids, cu, T = packed["input_ids"].cuda(), packed["cu_seqlens"], 50
    with torch.no_grad():
        with pytest.raises(ValueError, match="kv-cache"):
            m(input_ids=ids, cu_seqlens=cu, max_seqlen=30, use_cache=True)
        with pytest.raises(ValueError, match="kv-cache"):
            m(input_ids=ids, cu_seqlens=cu, max_seqlen=30, past_key_values=KVCache(2, 1, 64, 2, 64, "cuda"))
        with pytest.raises(ValueError, match="output_attentions"):
            m(input_ids=ids, cu_seqlens=cu, max_seqlen=30, output_attentions=True)
        m.config.log_attentions = True
        with pytest.raises(ValueError, match="log_attentions"):
            m(input_ids=ids, cu_seqlens=cu, max_seqlen=30)
        m.config.log_attentions = False
        mask = torch.ones(1, T, dtype=torch.long, device="cuda")
        mask[0, -3:] = 0
        with pytest.raises(ValueError, match="all ones"):
            m(input_ids=ids, cu_seqlens=cu, max_seqlen=30, attention_mask=mask)
        with pytest.raises(ValueError, match="number of packed tokens"):
            m(input_ids=ids, cu_seqlens=torch.tensor([0, 20, 49], dtype=torch.int32), max_seqlen=30)
        with pytest.raises(ValueError, match="one row"):
            m(input_ids=ids.view(2, 25), cu_seqlens=cu, max_seqlen=30)
        with pytest.raises(ValueError, match="max_seqlen"):
            m(input_ids=ids, cu_seqlens=cu, max_seqlen=29)
        # `cu_seqlens` alone is the right-padded collator's bookkeeping key and selects nothing
        assert torch.equal(m(input_ids=ids, cu_seqlens=cu).logits, m(input_ids=ids).logits)
        layer = m.model.layers[0]
        x = torch.zeros(1, T, 256, dtype=BF, device="cuda")
        with pytest.raises(ValueError, match="output_attentions"):
            layer(x, cu_seqlens=cu, max_seqlen=30, output_attentions=True)
        with pytest.raises(ValueError, match="kv-cache"):
            layer(x, cu_seqlens=cu, max_seqlen=30, past_key_value=(KVCache(2, 1, 64, 2, 64, "cuda"), 0))
        assert m(input_ids=ids, cu_seqlens=cu, max_seqlen=30, attention_mask=torch.ones_like(ids)).logits.shape == (1, T, 512)

"""Grouped-query attention on the GPU: the attention kernels with nkv < nh heads against fp32 eager attention with `repeat_kv`
(reference modeling_dreamllm.py:242-252, :357-379), bit for bit against the multi-head entry point on repeated K/V, and the GQA decoder
layer / causal LM against the reference's own GQA goldens (tests/golden/gqa_*.npz, oracle/gen_golden_gqa.py)."""
import glob
import math
import os

import numpy as np
import pytest
import torch

from oracle import decoder_oracle as O
from oracle import gqa_oracle as G
from oracle import gen_golden, gen_golden_gqa

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")
LAYERS = sorted(glob.glob(os.path.join(GOLDEN_DIR, "gqa_layer_*.npz")))


def _ref_core(q, k, v, causal, seqlens):
    """q [B,Sq,nh,d], k/v [B,Skv,nkv,d] -> out [B,Sq,nh*d]: the reference's eager math (:357-379) in the input dtype after `repeat_kv`,
    additive finfo.min mask (causal: top-left aligned, Sq == Skv), fp32 softmax cast back to the input dtype."""
    B, Sq, nh, d = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    dt = q.dtype
    qh = q.transpose(1, 2)
    kh, vh = (G.repeat_kv(t.transpose(1, 2), nh // nkv) for t in (k, v))
    w = torch.matmul(qh, kh.transpose(2, 3)) / math.sqrt(d)
    mask = torch.zeros(B, 1, Sq, Skv, dtype=dt)
    if causal:
        mask = mask.masked_fill(torch.ones(Sq, Skv, dtype=torch.bool).triu(1), torch.finfo(dt).min)
    if seqlens is not None:
        mask = mask.masked_fill((torch.arange(Skv)[None] >= seqlens[:, None])[:, None, None, :], torch.finfo(dt).min)
    w = torch.max(w + mask, torch.tensor(torch.finfo(dt).min, dtype=dt))
    p = torch.softmax(w, dim=-1, dtype=torch.float32).to(dt)
    return torch.matmul(p, vh).transpose(1, 2).reshape(B, Sq, nh * d)


def _views(buf, nh, nkv, d):
    """q [B,S,nh,d], k and v [B,S,nkv,d]: column-slice views of a fused [B, S, (nh + 2 nkv) d] projection buffer."""
    B, S = buf.shape[:2]
    return (buf[..., :nh * d].view(B, S, nh, d), buf[..., nh * d:(nh + nkv) * d].view(B, S, nkv, d),
            buf[..., (nh + nkv) * d:].view(B, S, nkv, d))


CASES = [
    # B, S, Skv, nh, nkv, d, causal, seqlens
    (2, 256, 256, 8, 4, 128, True, None),            # group 2
    (2, 200, 200, 8, 2, 128, True, [200, 77]),       # group 4, ragged: S not a tile multiple + right padding
    (2, 192, 192, 16, 2, 64, True, None),            # group 8, d 64
    (2, 320, 320, 8, 1, 64, True, [320, 129]),       # MQA, ragged
    (1, 300, 300, 4, 1, 128, False, None),           # MQA, non-causal
    (2, 128, 77, 8, 2, 64, False, None),             # non-causal cross-attention, Skv != S
    (1, 200, 333, 4, 2, 128, False, None),
]


@pytest.mark.parametrize("B,S,Skv,nh,nkv,d,causal,seqlens", CASES)
def test_gqa_kernels_vs_eager_repeat_kv(B, S, Skv, nh, nkv, d, causal, seqlens):
    from dreamllm_b200 import ops
    g = torch.Generator().manual_seed(1000 + S + nkv)
    q = torch.randn(B, S, nh, d, generator=g).to(BF)
    kv = torch.randn(B, Skv, 2, nkv, d, generator=g).to(BF)
    k, v = kv[:, :, 0], kv[:, :, 1]
    dout = (torch.randn(B, S, nh * d, generator=g) * 0.5).to(BF)
    sl = torch.tensor(seqlens) if seqlens is not None else None
    valid = torch.ones(B, S, dtype=torch.bool) if sl is None else (torch.arange(S)[None] < sl[:, None])
    dout = dout * valid[..., None]

    q32, k32, v32 = (t.float().requires_grad_(True) for t in (q, k, v))
    ref = _ref_core(q32, k32, v32, causal, sl)
    ref.backward(dout.float())
    qb, kb, vb = (t.clone().requires_grad_(True) for t in (q, k, v))
    refb = _ref_core(qb, kb, vb, causal, sl)
    refb.backward(dout)

    qd, kvd = q.cuda(), kv.cuda()
    kd, vd = kvd[:, :, 0], kvd[:, :, 1]
    sl_dev = sl.int().cuda() if sl is not None else None
    # self-attention reads q / k / v out of one fused [B, S, (nh + 2 nkv) d] buffer; the cross entry points take separate buffers
    fused = S == Skv and (causal or sl is not None)
    if fused:
        buf = torch.cat([q.reshape(B, S, -1), kv.reshape(B, S, -1)], -1).cuda()
        qd, kd, vd = _views(buf, nh, nkv, d)
        out, lse = ops.attn_fwd(qd, kd, vd, causal=causal, seqlens=sl_dev)
    else:
        out, lse = ops.attn_fwd_cross_lse(qd, kd, vd)
    torch.cuda.synchronize()
    o = out.cpu().float()
    assert float(o[~valid].abs().max() if (~valid).any() else 0.0) == 0.0
    torch.testing.assert_close(o[valid], ref.detach()[valid], rtol=2e-2, atol=2e-2)
    e_o = float((o[valid] - ref.detach()[valid]).abs().mean())
    e_r = float((refb.detach().float()[valid] - ref.detach()[valid]).abs().mean())
    assert e_o <= 1.5 * e_r + 1e-5, f"out: ours {e_o:.3e} vs reference-bf16 {e_r:.3e}"

    dq = torch.zeros_like(qd)
    dkv = torch.zeros(B, Skv, 2, nkv, d, device="cuda", dtype=BF)
    if fused:
        dbuf = torch.zeros_like(buf)
        dq, dk, dv = _views(dbuf, nh, nkv, d)
        ops.attn_bwd(dout.cuda(), qd, kd, vd, out, lse, dq, dk, dv, causal=causal, seqlens=sl_dev)
    else:
        dk, dv = dkv[:, :, 0], dkv[:, :, 1]
        ops.attn_bwd_cross(dout.cuda(), qd, kd, vd, out, lse, dq, dk, dv)
    torch.cuda.synchronize()
    for name, got, ref_g, refb_g in (("dq", dq, q32.grad, qb.grad), ("dk", dk, k32.grad, kb.grad), ("dv", dv, v32.grad, vb.grad)):
        gi = got.cpu().float()
        err = (gi - ref_g).abs()
        scale = ref_g.abs().max()
        assert float(err.max()) < 3e-2 * float(scale) + 1e-3, f"{name}: max err {float(err.max())} vs scale {float(scale)}"
        e_r = float((refb_g.float() - ref_g).abs().mean())
        assert float(err.mean()) <= 1.5 * e_r + 1e-5 * float(scale), f"{name}: ours {float(err.mean()):.3e} vs reference-bf16 {e_r:.3e}"
        if sl is not None:
            assert float(gi[~valid].abs().max()) == 0.0, f"{name} non-zero at padded positions"


@pytest.mark.parametrize("nh,nkv,d,causal,seqlens", [(8, 2, 128, True, None), (8, 1, 64, True, [384, 130]), (16, 4, 64, False, None)])
def test_gqa_bitwise_equals_mha_on_repeated_kv(nh, nkv, d, causal, seqlens):
    """Forward out / lse and dQ of the GQA path are bit-identical to the multi-head entry point run on K/V repeated to nh heads (the same
    tiles reach the same arithmetic); dK / dV, summed over the group inside one CTA, are bitwise repeatable."""
    from dreamllm_b200 import ops
    B, S = 2, 384
    gen = torch.Generator().manual_seed(77 + nkv)
    buf = torch.randn(B, S, (nh + 2 * nkv) * d, generator=gen).to(BF).cuda()
    q, k, v = _views(buf, nh, nkv, d)
    rep = torch.cat([q.reshape(B, S, -1), k.repeat_interleave(nh // nkv, 2).reshape(B, S, -1),
                     v.repeat_interleave(nh // nkv, 2).reshape(B, S, -1)], -1).contiguous()
    qm, km, vm = _views(rep, nh, nh, d)
    sl = torch.tensor(seqlens, dtype=torch.int32).cuda() if seqlens else None
    out, lse = ops.attn_fwd(q, k, v, causal=causal, seqlens=sl)
    out_m, lse_m = ops.attn_fwd(qm, km, vm, causal=causal, seqlens=sl)
    assert torch.equal(out, out_m) and torch.equal(lse, lse_m)
    dout = (torch.randn(B, S, nh * d, generator=gen) * 0.5).to(BF).cuda()
    grads = []
    for _ in range(2):
        dbuf = torch.full_like(buf, float("nan"))
        dq, dk, dv = _views(dbuf, nh, nkv, d)
        ops.attn_bwd(dout, q, k, v, out, lse, dq, dk, dv, causal=causal, seqlens=sl)
        grads.append(dbuf)
    dmb = torch.zeros_like(rep)
    dqm, dkm, dvm = _views(dmb, nh, nh, d)
    ops.attn_bwd(dout, qm, km, vm, out_m, lse_m, dqm, dkm, dvm, causal=causal, seqlens=sl)
    torch.cuda.synchronize()
    assert torch.equal(grads[0], grads[1])                                   # every column written (no NaN left) and repeatable
    assert not torch.isnan(grads[0]).any()
    assert torch.equal(_views(grads[0], nh, nkv, d)[0], dqm)
    dk, dv = _views(grads[0], nh, nkv, d)[1:]
    for got, want in ((dk, dkm), (dv, dvm)):                                  # the group sum of the per-q-head gradients
        want = want.float().view(B, S, nkv, nh // nkv, d).sum(3)
        torch.testing.assert_close(got.float(), want, rtol=2e-2, atol=2e-2 * float(want.abs().max()))


@pytest.mark.parametrize("masked", [False, True])
def test_gqa_kvcache_forward_bitwise_equals_mha(masked):
    from dreamllm_b200 import ops
    B, nh, nkv, d, max_len, past, Sq = 2, 8, 2, 128, 256, 150, 5
    gen = torch.Generator().manual_seed(5)
    kc = torch.zeros(B, max_len, nkv, d, dtype=BF)
    vc = torch.zeros(B, max_len, nkv, d, dtype=BF)
    kc[:, :past + Sq] = torch.randn(B, past + Sq, nkv, d, generator=gen).to(BF)
    vc[:, :past + Sq] = torch.randn(B, past + Sq, nkv, d, generator=gen).to(BF)
    q = torch.randn(B, Sq, nh, d, generator=gen).to(BF).cuda()
    kc, vc = kc.cuda(), vc.cuda()
    mask = None
    if masked:
        mask = torch.ones(B, 256, dtype=torch.uint8, device="cuda")
        mask[1, :40] = 0                                                       # left padding of row 1
    out = ops.attn_fwd_cache(q, kc, vc, past + Sq, causal=True, kv_mask=mask)
    rk, rv = (t.repeat_interleave(nh // nkv, 2).contiguous() for t in (kc, vc))
    out_m = ops.attn_fwd_cache(q, rk, rv, past + Sq, causal=True, kv_mask=mask)
    torch.cuda.synchronize()
    assert torch.equal(out, out_m)
    am = torch.ones(B, past + Sq, dtype=torch.long)
    if masked:
        am[1, :40] = 0
    qf, kf, vf = q.cpu().float(), kc[:, :past + Sq].cpu().float(), vc[:, :past + Sq].cpu().float()
    mask4 = O.causal_additive_mask_past(B, Sq, past, torch.float32, am)
    w = torch.matmul(qf.transpose(1, 2), G.repeat_kv(kf.transpose(1, 2), nh // nkv).transpose(2, 3)) / math.sqrt(d) + mask4
    ref = torch.matmul(torch.softmax(w, -1), G.repeat_kv(vf.transpose(1, 2), nh // nkv)).transpose(1, 2).reshape(B, Sq, nh * d)
    torch.testing.assert_close(out.cpu().float(), ref, rtol=2e-2, atol=2e-2)


def test_gqa_rejects_heads_not_divisible():
    from dreamllm_b200 import ops
    q = torch.zeros(1, 64, 6, 64, dtype=BF, device="cuda")
    k = torch.zeros(1, 64, 4, 64, dtype=BF, device="cuda")
    with pytest.raises(AssertionError, match="multiple of"):
        ops.attn_fwd_cross_lse(q, k, k)
    from dreamllm_b200._lib import lib
    L = lib()
    out = torch.empty(1, 64, 6 * 64, dtype=BF, device="cuda")
    lse = torch.empty(1, 6, 64, dtype=torch.float32, device="cuda")
    for nkv in (4, 0, -2):
        rc = L.dllm_attn_fwd_gqa(q.data_ptr(), k.data_ptr(), k.data_ptr(), out.data_ptr(), lse.data_ptr(), None, None, 0, 1, 64, 64, 64,
                                 6, nkv, 64, 6 * 64, 4 * 64, 6 * 64, 0, 0.125, torch.cuda.current_stream().cuda_stream)
        assert L.dllm_error_string(rc).decode() == "invalid shape / size", nkv


# ------------------------------------------------------------------------------------------------ decoder layer / model
def _err(a, ref):
    e = (a.float() - ref.float()).abs().flatten()
    k = max(1, int(e.numel() * 0.999))
    return float(e.mean()), float(e.kthvalue(k).values)


def _layer(hidden, inter, heads, kv_heads, p, theta=10000.0):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMDecoderLayer
    cfg = DreamLLMConfig(hidden_size=hidden, intermediate_size=inter, num_attention_heads=heads, num_key_value_heads=kv_heads,
                         num_hidden_layers=1, rope_theta=theta)
    layer = DreamLLMDecoderLayer(cfg)
    sd = {k: v.clone() for k, v in p.items()}
    sd["self_attn.rotary_emb.inv_freq"] = layer.self_attn.rotary_emb.inv_freq.clone()
    layer.load_state_dict(sd)
    return layer.to(device="cuda", dtype=BF)


@pytest.mark.parametrize("path", LAYERS, ids=[os.path.basename(p) for p in LAYERS])
def test_gqa_layer_vs_reference_golden(path):
    """The criteria of test_decoder_layer_gpu.py: as close to the reference's fp32 run as the reference's own bf16 run is."""
    g = np.load(path)
    hidden, inter, heads, bsz, seq, seed, pad = [int(v) for v in g["shape"]]
    kv_heads, theta = int(g["kv_heads"]), float(g["rope_theta"])
    rs, cs = [int(v) for v in g["stride"]]
    p = G.init_layer_params(hidden, inter, seed, heads, kv_heads)
    x, gy = gen_golden.make_inputs(hidden, bsz, seq, seed)
    am = gen_golden_gqa.pad_mask(bsz, seq, pad)
    valid = torch.ones(bsz, seq, dtype=torch.bool) if am is None else am.bool()
    if am is not None:
        gy = gy * am[..., None]

    pb = {k: v.to(BF).requires_grad_(True) for k, v in p.items()}
    xb = x.to(BF).requires_grad_(True)
    cos, sin = O.rope_tables(hidden // heads, 2048, base=theta, dtype=BF)
    pos = torch.arange(seq)[None].expand(bsz, -1)
    yb = G.decoder_layer(xb, pb, heads, kv_heads, cos, sin, pos, O.causal_additive_mask(bsz, seq, BF, am))
    yb.backward(gy.to(BF))

    layer = _layer(hidden, inter, heads, kv_heads, p, theta)
    xc = x.to(BF).cuda().requires_grad_(True)
    y = layer(xc, attention_mask=am.cuda() if am is not None else None)[0]
    y.backward(gy.to(BF).cuda())
    torch.cuda.synchronize()

    vs = valid[:, ::rs]
    sub = lambda t: t[:, ::rs, ::cs][vs]         # noqa: E731
    checks = [("y", sub(y.detach().cpu()), sub(yb.detach()), torch.from_numpy(g["y"])[vs]),
              ("dx", sub(xc.grad.cpu()), sub(xb.grad), torch.from_numpy(g["dx"])[vs])]
    for nm, ours_t, refb_t in (("y", y.detach().cpu(), yb.detach()), ("dx", xc.grad.cpu(), xb.grad)):
        want = float(g[nm + "_abs_sum"])          # whole-tensor |.| sums over the valid rows
        got, gotb = float(ours_t[valid].double().abs().sum()), float(refb_t[valid].double().abs().sum())
        assert abs(got - want) <= 2.0 * abs(gotb - want) + 2e-3 * want, (nm, got, gotb, want)
    ours_named = dict(layer.named_parameters())
    for k in O.LAYER_KEYS:
        gr, grb = ours_named[k].grad.cpu(), pb[k].grad
        sl = (lambda t: t[:8, :64]) if gr.dim() == 2 else (lambda t: t)
        checks.append(("d_" + k, sl(gr), sl(grb), torch.from_numpy(g["d_" + k])))
    report = []
    for name, ours, refb, gold in checks:
        m_o, p_o = _err(ours, gold)
        m_r, p_r = _err(refb, gold)
        scale = float(gold.abs().mean()) + 1e-12
        report.append(f"{name}: ours mean {m_o:.3e} p99.9 {p_o:.3e} | ref-bf16 mean {m_r:.3e} p99.9 {p_r:.3e} | |gold| {scale:.3e}")
        assert m_o <= 1.25 * m_r + 2e-3 * scale, report[-1]
        assert p_o <= 1.5 * p_r + 2e-2 * scale, report[-1]
    print("\n".join(report))
    for k in O.LAYER_KEYS:
        tot = float(ours_named[k].grad.double().sum())
        want = float(g["dsum_" + k])
        ref_tot = float(pb[k].grad.double().sum())
        assert abs(tot - want) <= 4.0 * abs(ref_tot - want) + 5e-2 * (abs(want) + 1e-3), (k, tot, want, ref_tot)


def test_gqa_cached_layer_vs_reference_golden():
    """The criteria of test_cached_layer_vs_oracle_left_padded_batch, against the reference's own GQA `past_key_value` run."""
    from dreamllm_b200.modeling_dreamllm import KVCache
    g = np.load(os.path.join(GOLDEN_DIR, "gqa_kvcache_layer.npz"))
    hidden, inter, heads, kv_heads = [int(v) for v in g["shape"]]
    p, calls = G.cached_decode_scenario(hidden, inter, heads, kv_heads)
    refbf = G.run_cached_scenario(p, calls, heads, kv_heads, BF)
    layer = _layer(hidden, inter, heads, kv_heads, p).eval()
    cache = KVCache(1, 2, 128, kv_heads, hidden // heads, "cuda")
    for i, (x, am, pos) in enumerate(calls):
        cache.set_mask(am.cuda())
        with torch.no_grad():
            y = layer(x.cuda().to(BF), position_ids=pos.cuda(), past_key_value=(cache, 0), use_cache=True)[0]
        cache.len += x.shape[1]
        valid = am[:, -x.shape[1]:].bool()
        r32 = torch.from_numpy(g[f"y{i}"])[valid]
        ours, rbf = y.cpu().float()[valid], refbf[i].float()[valid]
        e_o, e_r = float((ours - r32).abs().mean()), float((rbf - r32).abs().mean())
        assert e_o <= 1.5 * e_r + 1e-3 * float(r32.abs().mean()), (i, e_o, e_r)
        assert bool(torch.isfinite(y).all())
    # the cache holds the rotated keys of the kv heads only, as the reference's present key states (:355)
    k_final = torch.from_numpy(g["k_final"])                                   # [B, nkv, 4, d]
    ours_k = cache.k[0][:, cache.len - 4:cache.len].permute(0, 2, 1, 3).cpu().float()
    torch.testing.assert_close(ours_k, k_final, rtol=3e-2, atol=3e-2)


def _lm(kv_heads, layers=2, vocab=32008):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=vocab, hidden_size=512, intermediate_size=1024, num_hidden_layers=layers, num_attention_heads=8,
                         num_key_value_heads=kv_heads, max_position_embeddings=512)
    return DreamLLMForCausalMLM(cfg)


def test_gqa_causal_lm_decode_generate_and_cache_size():
    m = _lm(2).to(device="cuda", dtype=BF).eval()
    ids = torch.randint(0, 32000, (2, 70), device="cuda")
    with torch.no_grad():
        full = m(input_ids=ids).logits
        out = m(input_ids=ids[:, :50], use_cache=True)
        cache = out.past_key_values
        torch.testing.assert_close(out.logits, full[:, :50], rtol=2e-2, atol=2e-2)
        steps = [m(input_ids=ids[:, 50:64], past_key_values=cache, use_cache=True).logits]
        for t in range(64, 70):
            steps.append(m(input_ids=ids[:, t:t + 1], past_key_values=cache, use_cache=True).logits)
    inc = torch.cat(steps, 1)
    assert cache.len == 70
    torch.testing.assert_close(inc, full[:, 50:], rtol=2e-2, atol=3e-2)
    assert float((inc.argmax(-1) == full[:, 50:].argmax(-1)).float().mean()) > 0.97
    # KVCache bytes: 1 / group of the multi-head model's
    with torch.no_grad():
        mha_cache = _lm(8).to(device="cuda", dtype=BF).eval()(input_ids=ids[:, :8], use_cache=True).past_key_values
    nbytes = lambda c: sum(t.numel() * t.element_size() for t in c.k + c.v)        # noqa: E731
    assert nbytes(cache) * 4 == nbytes(mha_cache) and cache.k[0].shape[2] == 2
    # greedy ids == argmax of a full re-forward over the prefix (bf16 near-ties excepted)
    pr = ids[:, :33]
    gen = m.generate_greedy(pr, max_new_tokens=6)
    assert gen.shape == (2, 39) and torch.equal(gen[:, :33], pr)
    with torch.no_grad():
        for t in range(33, 39):
            ref = m(input_ids=gen[:, :t]).logits[:, -1]
            top2 = ref.topk(2).values
            sure = (top2[:, 0] - top2[:, 1]) > 0.05
            assert bool(((ref.argmax(-1) == gen[:, t]) | ~sure).all())
    # beam search over the GQA cache (repeat_interleave / reorder of the narrow K/V)
    beams = m.generate(pr, max_new_tokens=4, num_beams=3)
    assert beams.shape == (2, 37) and torch.equal(beams[:, :33], pr)


def test_gqa_fused_qkv_wgrad_lands_in_sharded_adamw_buckets(monkeypatch):
    """Under ShardedAdamW the fused q|k|v wgrad GEMM writes straight into the bucket: the narrower k/v blocks stay adjacent to q."""
    from dreamllm_b200 import modeling_dreamllm as MD
    from dreamllm_b200.zero import ShardedAdamW
    m = _lm(2, layers=3, vocab=512).to(device="cuda", dtype=BF).train()
    opt = ShardedAdamW(m.parameters(), lr=1e-3, bucket_cap_mb=0.5)
    assert len(opt.buckets) > 2
    seen = []
    real = MD.grad_out_view

    def spy(params):
        v = real(params)
        if len(params) == 3:
            seen.append(v)
        return v
    monkeypatch.setattr(MD, "grad_out_view", spy)
    ids = torch.randint(0, 512, (2, 96), generator=torch.Generator().manual_seed(3)).cuda()
    opt.zero_grad()
    m(input_ids=ids, labels=ids).loss.backward()
    torch.cuda.synchronize()
    assert len(seen) == 3 and all(v is not None for v in seen)
    for layer in m.model.layers:
        for p in (layer.self_attn.q_proj.weight, layer.self_attn.k_proj.weight, layer.self_attn.v_proj.weight):
            assert p.grad.data_ptr() == opt._bucket_of[p].gviews[p].data_ptr()
    opt.step()


def test_gqa_checkpointed_recompute_is_bitwise_repeatable():
    def run(ckpt):
        m = _lm(2, layers=3, vocab=512).to(device="cuda", dtype=BF).train()
        if ckpt:
            m.gradient_checkpointing_enable()
        ids = torch.randint(1, 512, (2, 160), generator=torch.Generator().manual_seed(1)).cuda()
        mask = torch.ones_like(ids)
        mask[1, 100:] = 0
        labels = ids.masked_fill(mask == 0, -100)
        out = m(input_ids=ids, attention_mask=mask, labels=labels)
        out.loss.backward()
        return out.loss.detach(), {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    l0, g0 = run(False)
    l1, g1 = run(True)
    l2, g2 = run(True)
    assert torch.equal(l1, l2) and abs(float(l0) - float(l1)) <= 1e-5 * abs(float(l0))
    for k in g0:
        assert torch.equal(g1[k], g2[k]), k                                    # recompute inside backward: bitwise repeatable
        torch.testing.assert_close(g1[k].float(), g0[k].float(), rtol=1e-3, atol=1e-6, msg=k)
    p = G.init_layer_params(512, 1024, 4, 8, 2)
    layer = _layer(512, 1024, 8, 2, p)
    x = torch.randn(1, 200, 512, device="cuda").to(BF)
    assert torch.equal(layer(x)[0], layer(x)[0])

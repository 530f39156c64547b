"""wgmma flash attention (fwd + two-kernel bwd) vs the CPU oracle's eager softmax(QK^T/sqrt(d)+mask)V
(oracle.decoder_oracle.attention_eager's core, reference modeling_dreamllm.py:357-379) on seeded inputs."""
import math

import pytest
import torch

from oracle import decoder_oracle as O

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _ref_core(q, k, v, causal, seqlens):
    """q,k,v: [B,S,nh,d] fp32 or bf16 -> out [B,S,nh*d]; eager math exactly as the reference (:357-379): scores in the input dtype,
    additive finfo.min mask, clamp, fp32 softmax cast back to the input dtype (:378), PV in the input dtype.  Run in bf16 it IS the
    reference's bf16 eager path — the like-for-like yardstick for our bf16 kernels."""
    B, S, nh, d = q.shape
    dt = q.dtype
    qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))
    w = torch.matmul(qh, kh.transpose(2, 3)) / math.sqrt(d)
    am = None
    if seqlens is not None:
        am = (torch.arange(S)[None] < seqlens[:, None]).long()
    if causal:
        mask = O.causal_additive_mask(B, S, dt, am)
    else:
        mask = torch.zeros(B, 1, S, S, dtype=dt)
        if am is not None:
            mask = mask.masked_fill((am == 0)[:, None, None, :], torch.finfo(dt).min)
    w = torch.max(w + mask, torch.tensor(torch.finfo(dt).min, dtype=dt))
    p = torch.softmax(w, dim=-1, dtype=torch.float32).to(dt)
    return torch.matmul(p, vh).transpose(1, 2).reshape(B, S, nh * d)


CASES = [
    # B, S, nh, d, causal, seqlens
    (1, 128, 1, 128, True, None),
    (2, 512, 2, 128, True, None),
    (2, 200, 3, 128, True, [200, 77]),       # ragged: S not a tile multiple + right padding
    (1, 577, 2, 64, False, None),            # CLIP-like: non-causal, d=64, 577 tokens
    (2, 320, 2, 64, True, [320, 129]),
    (1, 1024, 2, 128, False, None),
]


@pytest.mark.parametrize("B,S,nh,d,causal,seqlens", CASES)
def test_attn_fwd_bwd_vs_oracle(B, S, nh, d, causal, seqlens):
    from dreamllm_b200 import ops

    g = torch.Generator().manual_seed(100 + S)
    qkv = torch.randn(B, S, 3, nh, d, generator=g).to(BF)
    dout = (torch.randn(B, S, nh * d, generator=g) * 0.5).to(BF)
    sl = torch.tensor(seqlens) if seqlens is not None else None
    valid = torch.ones(B, S, dtype=torch.bool) if sl is None else (torch.arange(S)[None] < sl[:, None])
    dout = dout * valid[..., None]            # padded positions carry no loss

    q32, k32, v32 = (qkv[:, :, i].float().requires_grad_(True) for i in range(3))
    ref = _ref_core(q32, k32, v32, causal, sl)
    ref.backward(dout.float())
    # the reference's own bf16 path on the same inputs: how far bf16 arithmetic alone moves the result
    qb, kb, vb = (qkv[:, :, i].clone().requires_grad_(True) for i in range(3))
    refb = _ref_core(qb, kb, vb, causal, sl)
    refb.backward(dout)

    dev = qkv.cuda()
    q, k, v = dev[:, :, 0], dev[:, :, 1], dev[:, :, 2]
    sl_dev = sl.int().cuda() if sl is not None else None
    out, lse = ops.attn_fwd(q, k, v, causal=causal, seqlens=sl_dev)
    torch.cuda.synchronize()
    o = out.cpu().float()
    # pad rows: reference flash path re-inserts zeros (pad_input); eager path differs there -> compare valid rows only
    assert float(o[~valid].abs().max() if (~valid).any() else 0.0) == 0.0
    torch.testing.assert_close(o[valid], ref.detach()[valid], rtol=2e-2, atol=2e-2)
    # like-for-like (DESIGN.md §2): our bf16 error vs the fp32 reference is bounded by the reference's own bf16 error vs fp32
    e_o = float((o[valid] - ref.detach()[valid]).abs().mean())
    e_r = float((refb.detach().float()[valid] - ref.detach()[valid]).abs().mean())
    assert e_o <= 1.5 * e_r + 1e-5, f"out: ours {e_o:.3e} vs reference-bf16 {e_r:.3e}"

    dqkv = torch.zeros_like(dev)
    ops.attn_bwd(dout.cuda(), q, k, v, out, lse, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], causal=causal, seqlens=sl_dev)
    torch.cuda.synchronize()
    got = dqkv.cpu().float()
    for i, (name, ref_g, refb_g) in enumerate((("dq", q32.grad, qb.grad), ("dk", k32.grad, kb.grad), ("dv", v32.grad, vb.grad))):
        gi = got[:, :, i]
        err = (gi - ref_g).abs()
        scale = ref_g.abs().max()
        assert float(err.max()) < 3e-2 * float(scale) + 1e-3, f"{name}: max err {float(err.max())} vs scale {float(scale)}"
        e_r = float((refb_g.float() - ref_g).abs().mean())
        assert float(err.mean()) <= 1.5 * e_r + 1e-5 * float(scale), f"{name}: ours {float(err.mean()):.3e} vs reference-bf16 {e_r:.3e}"
        if sl is not None:
            assert float(gi[~valid].abs().max()) == 0.0, f"{name} non-zero at padded positions"


def test_attn_full_size_properties():
    """C2 shape (B=8,S=2048,nh=32,d=128): too big for the CPU oracle -> size-independent properties.
    (1) rows of softmax sum to 1: with V = ones, out == 1;  (2) causality: perturbing the last 512 tokens' k/v
    leaves the first 1536 outputs bit-identical;  (3) spot-check 2 (b,h) pairs against the oracle."""
    from dreamllm_b200 import ops

    B, S, nh, d = 8, 2048, 32, 128
    g = torch.Generator(device="cuda").manual_seed(7)
    qkv = torch.randn(B, S, 3, nh, d, device="cuda", generator=g).to(BF)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    out, lse = ops.attn_fwd(q, k, v)
    ones = qkv.clone()
    ones[:, :, 2] = 1.0
    out1, _ = ops.attn_fwd(ones[:, :, 0], ones[:, :, 1], ones[:, :, 2])
    torch.testing.assert_close(out1.float(), torch.ones_like(out1).float(), rtol=0, atol=8e-3)
    pert = qkv.clone()
    pert[:, 1536:, 1:] += 1.0
    out2, _ = ops.attn_fwd(pert[:, :, 0], pert[:, :, 1], pert[:, :, 2])
    assert torch.equal(out2[:, :1536], out[:, :1536])
    for (b, h) in ((0, 0), (7, 31)):
        qs, ks, vs = (qkv[b:b + 1, :, i, h:h + 1].cpu().float() for i in range(3))
        ref = _ref_core(qs, ks, vs, True, None)
        torch.testing.assert_close(out[b:b + 1, :, h * d:(h + 1) * d].cpu().float(), ref, rtol=2e-2, atol=2e-2)

"""One-token decode step: `attn_decode` (split-KV attention reading the cache length from the device), `rope_append_kv`, the captured
`DecodeGraph` step and `generate(use_cuda_graph=True)`.

`attn_decode` is checked against a float64 restatement of its own algorithm that rounds to bf16 where the kernel does (the exp2 weights
before P.V, the output): each split walks its 64-key chunks with a running max and sum, and the split partials are merged in fixed
order.  So the bound is the tower-kernel one: bf16 outputs within 1 ulp of the rounded float64 result, at most 1 % of the
elements differ at all; the kernel's exp2 and dot products run in fp32, so a weight whose bf16 rounding sits at a tie can round the
other way, and in an output that is a cancellation that moves it by more than 1 ulp: such outputs (at most 0.1 %) are held to one
rounding step of the weights instead.  The like-for-like bound of DESIGN.md §2 against `attn_fwd_cache` on the same inputs is checked
as well."""
import math

import pytest
import torch

from oracle import decoder_oracle as O
from oracle import gqa_oracle as G

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
LOG2E = 1.4426950408889634


def _ops():
    from dreamllm_b200 import ops
    return ops


def _ref_decode(q, K, V, kv_len, mask, split_len, scale):
    """float64 attn_decode: q [B, nh, d], K/V [B, max_len, nkv, d] (CPU), keys [0, kv_len).  Returns float64 [B, nh * d] before rounding
    and the L1 mass sum(P |V|) / l of every output (what one bf16 rounding step of the weights can move it by, times 2^-8)."""
    B, nh, d = q.shape
    nkv = K.shape[2]
    g = nh // nkv
    c = float(torch.tensor(scale * LOG2E, dtype=torch.float32))         # the kernel's fp32 scale * log2(e)
    n_split = (kv_len + split_len - 1) // split_len
    cps = split_len // 64
    Lp = n_split * split_len
    qd = q.double().view(B, nkv, g, d)
    Kd = torch.zeros(B, Lp, nkv, d, dtype=torch.float64)
    Vd = torch.zeros(B, Lp, nkv, d, dtype=torch.float64)
    Kd[:, :kv_len], Vd[:, :kv_len] = K[:, :kv_len].double(), V[:, :kv_len].double()
    s = torch.einsum("bkgd,blkd->bkgl", qd, Kd)                           # [B, nkv, g, Lp]
    ok = torch.arange(Lp) < kv_len
    ok = ok[None].expand(B, Lp).clone()
    if mask is not None:
        ok[:, :kv_len] &= mask[:, :kv_len].bool()
    s = s.masked_fill(~ok[:, None, None, :], float("-inf")) * c
    s = s.view(B, nkv, g, n_split, cps, 64)                               # key = split * split_len + chunk * 64 + i
    Vc = Vd.view(B, n_split, cps, 64, nkv, d)
    m = torch.full((B, nkv, g, n_split), float("-inf"), dtype=torch.float64)
    l = torch.zeros_like(m)
    o = torch.zeros(B, nkv, g, n_split, d, dtype=torch.float64)
    oa = torch.zeros_like(o)
    for j in range(cps):
        sj = s[:, :, :, :, j]                                             # [B, nkv, g, n_split, 64]
        m_new = torch.maximum(m, sj.amax(-1))
        alpha = torch.where(m == float("-inf"), torch.zeros_like(m), torch.exp2(m - m_new))
        m_use = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
        p = torch.exp2(sj - m_use[..., None])
        l = l * alpha + p.sum(-1)
        pb = p.to(torch.float32).to(BF).double()
        o = o * alpha[..., None] + torch.einsum("bkgsi,bsikd->bkgsd", pb, Vc[:, :, j])
        oa = oa * alpha[..., None] + torch.einsum("bkgsi,bsikd->bkgsd", pb, Vc[:, :, j].abs())
        m = m_new
    M = m.amax(-1, keepdim=True)
    w = torch.where(m == float("-inf"), torch.zeros_like(m), torch.exp2(m - torch.where(M == float("-inf"), torch.zeros_like(M), M)))
    lt = (w * l).sum(-1)
    ot = (w[..., None] * o).sum(-2)
    inv = torch.where(lt > 0, 1.0 / lt.clamp_min(1e-300), torch.zeros_like(lt))[..., None]
    return (ot * inv).reshape(B, nh * d), ((w[..., None] * oa).sum(-2) * inv).reshape(B, nh * d)


def _ulps(got_bf, ref64):
    """|got - bf16(ref)| in units of the bf16 spacing at bf16(ref) (2^(e - 8) for |r| = m 2^e, m in [0.5, 1))."""
    r = ref64.to(torch.float32).to(BF).float()
    _, e = torch.frexp(r)
    spacing = torch.where(r != 0, torch.ldexp(torch.ones_like(r), e - 8), torch.full_like(r, 2.0 ** -133))
    return (got_bf.float() - r).abs() / spacing


def _inputs(B, nh, nkv, d, max_len, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, nh, d, generator=g).to(BF)
    K = torch.randn(B, max_len, nkv, d, generator=g).to(BF)
    V = torch.randn(B, max_len, nkv, d, generator=g).to(BF)
    return q, K, V


def _left_pad_mask(B, max_len, kv_len):
    ld = (max_len + 63) // 64 * 64
    mask = torch.ones(B, ld, dtype=torch.uint8)
    for b in range(1, B, 2):                                              # odd rows: a left-padded prompt
        mask[b, :min(kv_len - 1, 5 + 17 * b)] = 0
    return mask


MAX_LEN = 520


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("nkv", [32, 8, 4])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_attn_decode_vs_float64(d, nkv, B):
    ops = _ops()
    nh = 32
    q, K, V = _inputs(B, nh, nkv, d, MAX_LEN, 1000 + d + nkv + B)
    qd, Kd, Vd = q.cuda(), K.cuda(), V.cuda()
    scale = d ** -0.5
    # the device's own plan, and a plan forced to 64-row splits (many SMs): both cut the cache at split boundaries
    for sms in (0, 1 << 20):
        ns, sl = ops.attn_decode_plan(B, nkv, MAX_LEN, sms)
        bounds = sorted({x for s in range(1, ns) for x in (s * sl - 1, s * sl, s * sl + 1)} & set(range(1, MAX_LEN + 1)))
        lens = sorted({1, 63, 64, 65, 127, 128, 129, MAX_LEN} | set(bounds[:9]))
        for kv_len in lens:
            for masked in (False, True):
                mask = _left_pad_mask(B, MAX_LEN, kv_len) if masked else None
                kvl = torch.tensor([kv_len], dtype=torch.int32, device="cuda")
                out = ops.attn_decode(qd, Kd, Vd, kvl, kv_mask=None if mask is None else mask.cuda(), sms=sms).cpu()
                ref, mass = _ref_decode(q, K, V, kv_len, mask, sl, scale)
                u = _ulps(out, ref)
                tag = (sms, kv_len, masked)
                assert float((u > 0).float().mean()) <= 0.01, (tag, float((u > 0).float().mean()))
                assert float((u > 1).float().mean()) <= 0.001, (tag, float((u > 1).float().mean()))
                # beyond 1 ulp only where a weight's bf16 rounding flipped (fp32 vs float64 exp2 at a rounding tie) inside an output
                # that is a cancellation: at most one rounding step of the weights, 2^-8 of the L1 mass
                err = (out.double() - ref.float().to(BF).double()).abs()
                assert bool((err[u > 1] <= 2.0 ** -8 * mass[u > 1]).all()), tag
                if kv_len in (129, MAX_LEN):
                    # like-for-like: our error vs exact attention within 1.5x attn_fwd_cache's on the same inputs
                    exact = torch.einsum("bhl,blhd->bhd", torch.softmax(
                        torch.einsum("bhd,blhd->bhl", q.double(), K[:, :kv_len].double().repeat_interleave(nh // nkv, 2)) * scale
                        + (0 if mask is None else torch.where(mask[:, None, :kv_len].bool(), 0.0, float("-inf"))), -1),
                        V[:, :kv_len].double().repeat_interleave(nh // nkv, 2)).reshape(B, nh * d)
                    fc = ops.attn_fwd_cache(qd.view(B, 1, nh, d), Kd, Vd, kv_len, causal=True,
                                            kv_mask=None if mask is None else mask.cuda()).view(B, nh * d).cpu()
                    e_o = float((out.double() - exact).abs().mean())
                    e_r = float((fc.double() - exact).abs().mean())
                    assert e_o <= 1.5 * e_r + 1e-6, (tag, e_o, e_r)


def test_attn_decode_deterministic_and_blind_past_kv_len():
    ops = _ops()
    B, nh, nkv, d, max_len, kv_len = 3, 32, 8, 128, 1024, 333
    q, K, V = (t.cuda() for t in _inputs(B, nh, nkv, d, max_len, 7))
    kvl = torch.tensor([kv_len], dtype=torch.int32, device="cuda")
    mask = _left_pad_mask(B, max_len, kv_len).cuda()
    a = ops.attn_decode(q, K, V, kvl, kv_mask=mask)
    b = ops.attn_decode(q, K, V, kvl, kv_mask=mask)
    assert torch.equal(a, b)
    K2, V2 = K.clone(), V.clone()
    K2[:, kv_len:] = 1000.0
    V2[:, kv_len:] = -3.0e4
    assert torch.equal(ops.attn_decode(q, K2, V2, kvl, kv_mask=mask), a)
    # the same kv_len through a plan made for a longer cache: the split length depends on (B, nkv, SMs) only
    big = 4096
    Kb = torch.zeros(B, big, nkv, d, dtype=BF, device="cuda")
    Vb = torch.zeros_like(Kb)
    Kb[:, :max_len], Vb[:, :max_len] = K, V
    maskb = torch.ones(B, big, dtype=torch.uint8, device="cuda")
    maskb[:, :mask.shape[1]] = mask
    assert ops.attn_decode_plan(B, nkv, big)[0] > ops.attn_decode_plan(B, nkv, max_len)[0]
    assert torch.equal(ops.attn_decode(q, Kb, Vb, kvl, kv_mask=maskb), a)


@pytest.mark.parametrize("d,nh,nkv", [(128, 32, 8), (64, 4, 4)])
def test_rope_append_kv_matches_rope_and_copies(d, nh, nkv):
    ops = _ops()
    B, max_len, row = 5, 96, 41
    g = torch.Generator().manual_seed(11)
    qkv = torch.randn(B, (nh + 2 * nkv) * d, generator=g).to(BF).cuda()
    cos, sin = (t.to(BF).cuda() for t in O.rope_tables(d, 2048))
    pos = torch.tensor([41, 3, 0, 40, 17], dtype=torch.int32, device="cuda")     # left-padded rows sit at different positions
    kc = torch.randn(B, max_len, nkv, d, generator=g).to(BF).cuda()
    vc = torch.randn(B, max_len, nkv, d, generator=g).to(BF).cuda()
    ref_qkv, ref_k, ref_v = qkv.clone(), kc.clone(), vc.clone()
    ops.rope_(ref_qkv, cos, sin, pos, nh + nkv, d)
    ref_k[:, row] = ref_qkv[:, nh * d:(nh + nkv) * d].view(B, nkv, d)
    ref_v[:, row] = ref_qkv[:, (nh + nkv) * d:].view(B, nkv, d)
    ops.rope_append_kv_(qkv, cos, sin, pos, kc, vc, torch.tensor([row], dtype=torch.int32, device="cuda"), nh, nkv, d)
    assert torch.equal(qkv[:, :(nh + nkv) * d], ref_qkv[:, :(nh + nkv) * d])
    assert torch.equal(kc, ref_k) and torch.equal(vc, ref_v)


# ------------------------------------------------------------------------------------------------ captured step and generate
def _model(hidden, heads, kv_heads, layers, vocab=512, seed=7, head_scale=8.0):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    cfg = DreamLLMConfig(vocab_size=vocab, hidden_size=hidden, intermediate_size=2 * hidden, num_hidden_layers=layers,
                         num_attention_heads=heads, num_key_value_heads=kv_heads, max_position_embeddings=256)
    torch.manual_seed(seed)
    model = DreamLLMForCausalMLM(cfg)
    with torch.no_grad():                                  # N(0, 0.02) init gives near-uniform logits; widen the head so margins are real
        model.lm_head.weight.mul_(head_scale)
    return model.to(device="cuda", dtype=BF).eval()


MODELS = [  # hidden, heads, kv heads, layers  (d = hidden / heads)
    (256, 2, 2, 2),      # MHA, d 128
    (256, 4, 1, 3),      # GQA group 4, d 64
    (512, 8, 4, 2),      # GQA group 2, d 64
    (512, 4, 4, 4),      # MHA, d 128
]


def _mask_kw(am):
    return {} if am is None else dict(attention_mask=am, position_ids=(am.long().cumsum(-1) - 1).masked_fill(am == 0, 1))


@pytest.mark.parametrize("hidden,heads,kv_heads,layers", [MODELS[0], MODELS[1]])
def test_decode_graph_replay_equals_eager(hidden, heads, kv_heads, layers):
    """Replay == eager step, bit for bit, logits and caches, over 16 tokens of a left-padded batch whose rows are re-ordered (as beam
    search does, K/V and padding mask in place) between steps."""
    from dreamllm_b200.decode import DecodeGraph
    model = _model(hidden, heads, kv_heads, layers)
    B, S = 3, 40
    ids = torch.randint(0, 512, (B, S), generator=torch.Generator().manual_seed(5)).cuda()
    am = torch.ones(B, S, dtype=torch.long, device="cuda")
    am[1, :9] = 0
    am[2, :23] = 0
    caches = []
    for _ in range(2):
        with torch.no_grad():
            caches.append(model(input_ids=ids, use_cache=True, last_token_logits_only=True, **_mask_kw(am)).past_key_values)
    assert caches[0].mask is not None
    pos = am.sum(-1)
    eager, graph = DecodeGraph(model, caches[0], B, positions=pos), DecodeGraph(model, caches[1], B, positions=pos)
    feed = torch.randint(0, 512, (16, B), generator=torch.Generator().manual_seed(6)).cuda()
    perms = [torch.randperm(B, generator=torch.Generator().manual_seed(100 + t)).cuda() for t in range(16)]
    for t in range(16):
        if t % 3 == 2:                                                    # rows take another row's history (and its mask row)
            for c, dg in ((caches[0], eager), (caches[1], graph)):
                c.reorder(perms[t])
                dg.pos.copy_(dg.pos[perms[t]])
        eager.ids.copy_(feed[t])
        graph.ids.copy_(feed[t])
        a = eager.step().clone()
        b = graph.replay().clone()
        assert torch.equal(a, b), t
    assert caches[0].len == caches[1].len == S + 16
    assert torch.equal(caches[0].mask, caches[1].mask) and not bool(caches[0].mask[:, :S].all())
    for li in range(layers):
        assert torch.equal(caches[0].k[li], caches[1].k[li]) and torch.equal(caches[0].v[li], caches[1].v[li])


def _oracle_logits(model, x, am, dtype):
    """Logits of every position from the CPU oracle (oracle/gqa_oracle.py decoder layers) in `dtype`, starting from the input embeddings
    x [B, L, H] (bf16: the token embeddings, with the image features spliced in where the prompt has them); positions and key masking
    from the left-padding mask `am` [B, L] (None: no padding), as the kv-cache path takes them."""
    cfg = model.config
    heads = cfg.num_attention_heads
    kv_heads = getattr(cfg, "num_key_value_heads", None) or heads
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items() if k.startswith(("model.layers.", "model.norm.", "lm_head."))}
    B, L, H = x.shape
    x = x.to(dtype)
    cos, sin = O.rope_tables(H // heads, 2048, dtype=dtype)
    if am is None:
        pos = torch.arange(L)[None].expand(B, -1)
    else:
        pos = (am.long().cumsum(-1) - 1).masked_fill(am == 0, 1)
    mask = O.causal_additive_mask(B, L, dtype, am)
    with torch.no_grad():
        for i in range(cfg.num_hidden_layers):
            p = {k: sd[f"model.layers.{i}.{k}"].to(dtype) for k in O.LAYER_KEYS}
            x = G.decoder_layer(x, p, heads, kv_heads, cos, sin, pos, mask)
        return torch.nn.functional.linear(O.rmsnorm(x, sd["model.norm.weight"].to(dtype)), sd["lm_head.weight"].to(dtype)).float()


def _graph_greedy(model, ids, n_new, am=None, images=None):
    """Greedy decoding through the DecodeGraph: (ids + n_new tokens [B, S + n_new], the logits that picked them [B, n_new, V] (the first
    from the prefill), the prefill's input embeddings [B, S, H])."""
    from dreamllm_b200.decode import DecodeGraph
    with torch.no_grad():
        out = model(input_ids=ids, images=images, use_cache=True, last_token_logits_only=True, **_mask_kw(am))
        x0 = model.model(input_ids=ids, images=images, output_hidden_states=True, **_mask_kw(am)).hidden_states[0]
    dg = DecodeGraph(model, out.past_key_values, ids.shape[0], positions=None if am is None else am.long().sum(-1))
    logits = [out.logits[:, -1]]
    toks = [logits[-1].argmax(-1)]
    for _ in range(n_new - 1):
        dg.ids.copy_(toks[-1])
        logits.append(dg.replay().clone())
        toks.append(logits[-1].argmax(-1))
    return torch.cat([ids, torch.stack(toks, 1)], 1), torch.stack(logits, 1).cpu(), x0.cpu()


def _check_margin_rule(model, ids, seq, lg, x0, eager, am=None):
    """test_causal_lm_gpu's rule on the decoded positions, against the oracle run over the graph path's own sequence:
      * budget e = 2 x max|logits(oracle bf16) - logits(oracle fp32)|;
      * the graph path's logits (the same positions, through the kv-cache) stay within e of the fp32 oracle's;
      * most decoded positions have a top-1 margin > 2e (otherwise the rule is vacuous), and while every decoded position so far is
        such a clear one, the graph path, the eager path and the fp32 oracle pick the same id.
    Returns the number of positions compared (the callers ask for at least two per row on average; the majority rule above is what
    keeps the check from being vacuous)."""
    B, S = ids.shape
    n = lg.shape[1]
    emb = model.model.embed_tokens.weight.detach().cpu()
    x = torch.cat([x0, emb[seq[:, S:S + n - 1].cpu()]], 1)
    am_full = None if am is None else torch.cat([am.cpu(), torch.ones(B, n - 1, dtype=am.dtype)], 1)
    l32 = _oracle_logits(model, x, am_full, torch.float32)[:, S - 1:]
    lbf = _oracle_logits(model, x, am_full, BF)[:, S - 1:]
    budget = 2.0 * float((lbf - l32).abs().max())
    err = float((lg - l32).abs().max())
    assert err <= budget, (err, budget)
    top2 = l32.topk(2, -1).values
    clear = (top2[..., 0] - top2[..., 1]) > 2 * budget
    assert float(clear.float().mean()) > 0.5, f"only {float(clear.float().mean()):.2f} of the decoded positions have a clear margin"
    alive = torch.cumprod(clear.long(), 1).bool()
    pick = l32.argmax(-1)
    assert torch.equal(seq.cpu()[:, S:S + n][alive], pick[alive])
    assert torch.equal(eager.cpu()[:, S:S + n][alive], pick[alive])
    return int(alive.sum())


@pytest.mark.parametrize("hidden,heads,kv_heads,layers", MODELS)
def test_generate_with_cuda_graph(hidden, heads, kv_heads, layers):
    model = _model(hidden, heads, kv_heads, layers)
    B, S, n_new = 8, 24, 12
    ids = torch.randint(0, 512, (B, S), generator=torch.Generator().manual_seed(8)).cuda()
    seq, lg, x0 = _graph_greedy(model, ids, n_new)
    assert torch.equal(model.generate(ids, max_new_tokens=n_new, use_cuda_graph=True), seq)
    eager = model.generate(ids, max_new_tokens=n_new)
    assert _check_margin_rule(model, ids, seq, lg, x0, eager) >= 2 * B


def test_generate_with_cuda_graph_image_prompt():
    """A prompt with an image: the prefill runs CLIP and the image splice, then the decode steps replay the graph."""
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    from dreamllm_b200.modeling_plugins import CLIPVisionEmbedding, DreamEmbedding
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=32008, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                         max_position_embeddings=256)
    m = DreamLLMForCausalMLM(cfg)
    with torch.no_grad():
        m.lm_head.weight.mul_(8.0)
    clip = CLIPVisionEmbedding(dict(hidden_size=256, intermediate_size=512, num_hidden_layers=3, num_attention_heads=4, image_size=56,
                                    patch_size=14), embed_hidden_size=256)
    m.model.attach_plugins(clip, DreamEmbedding(num_dream_queries=8, embed_hidden_size=256), image_start_id=32003, dream_start_id=32006)
    m = m.to(device="cuda", dtype=BF).eval()
    P = clip.embed_len
    B, n_new = 2, 10
    text = torch.randint(3, 32000, (B, 8), generator=torch.Generator().manual_seed(4))
    ids = torch.cat([torch.tensor([[1, 32003] + [32002] * P + [32004]] * B), text], 1).cuda()
    imgs = torch.randn(B, 3, 56, 56, generator=torch.Generator().manual_seed(5)).to(BF).cuda()
    seq, lg, x0 = _graph_greedy(m, ids, n_new, images=imgs)
    assert not torch.equal(x0[:, 2:2 + P], m.model.embed_tokens.weight.detach().cpu()[ids[:, 2:2 + P].cpu()])   # CLIP features spliced
    assert torch.equal(m.generate(ids, images=imgs, max_new_tokens=n_new, use_cuda_graph=True), seq)
    eager = m.generate(ids, images=imgs, max_new_tokens=n_new)
    assert _check_margin_rule(m, ids, seq, lg, x0, eager) >= 2 * B


def test_generate_with_cuda_graph_batches_and_controls():
    model = _model(512, 8, 4, 2)
    dev = "cuda"
    B, S = 3, 30
    ids = torch.randint(3, 512, (B, S), generator=torch.Generator().manual_seed(9)).to(dev)
    am = torch.ones(B, S, dtype=torch.long, device=dev)
    am[1, :7] = 0
    am[2, :19] = 0                                                        # left padding
    seq, lg, x0 = _graph_greedy(model, ids, 10, am=am)
    assert torch.equal(model.generate(ids, attention_mask=am, max_new_tokens=10, use_cuda_graph=True), seq)
    eager = model.generate(ids, attention_mask=am, max_new_tokens=10)
    assert _check_margin_rule(model, ids, seq, lg, x0, eager, am=am) >= 2 * B
    # EOS + pad filling, stopping criteria, seeded sampling: identical control flow to the eager loop
    free = seq[0, S:S + 8].tolist()
    eos = free[2]
    k = free.index(eos)
    out = model.generate(ids, attention_mask=am, max_new_tokens=8, eos_token_id=eos, pad_token_id=1, use_cuda_graph=True)
    row = out[0, S:].tolist()
    assert row[:k + 1] == free[:k + 1] and all(t == 1 for t in row[k + 1:])
    calls = []

    def crit(seq, scores):
        calls.append(scores.shape)
        return seq.shape[1] >= S + 4

    out = model.generate(ids, attention_mask=am, max_new_tokens=10, stopping_criteria=[crit], use_cuda_graph=True)
    assert out.shape[1] == S + 4 and calls[0] == (B, 512)

    def sample():
        return model.generate(ids, attention_mask=am, max_new_tokens=8, do_sample=True, top_k=20, temperature=0.8,
                              generator=torch.Generator(device=dev).manual_seed(3), use_cuda_graph=True)

    assert torch.equal(sample(), sample())


@pytest.mark.parametrize("padded", [False, True])
def test_beam_search_with_cuda_graph(padded):
    """beam_search(num_beams=5): the cache is repeated per beam before the graph is built and re-ordered in place (K/V and, for a
    left-padded batch, the padding mask) between replays.  Every generated token equals the eager beam search's, and the best
    hypotheses' scores (mean log-probability of the generated tokens) agree within the logits budget of the margin rule."""
    from dreamllm_b200.generation import beam_search
    model = _model(512, 8, 4, 2)
    B, S, n_new = 2, 30, 10
    ids = torch.randint(3, 512, (B, S), generator=torch.Generator().manual_seed(12)).cuda()
    am = None
    if padded:
        am = torch.ones(B, S, dtype=torch.long, device="cuda")
        am[1, :11] = 0
    x0 = model.model.embed_tokens.weight.detach().cpu()[ids.cpu()]
    am_cpu = None if am is None else am.cpu()
    budget = 2.0 * float((_oracle_logits(model, x0, am_cpu, BF) - _oracle_logits(model, x0, am_cpu, torch.float32)).abs().max())
    kw = dict(num_beams=5, max_new_tokens=n_new, attention_mask=am, return_scores=True)
    seq_e, sc_e = beam_search(model, ids, **kw)
    seq_g, sc_g = beam_search(model, ids, use_cuda_graph=True, **kw)
    assert seq_e.shape[1] == S + n_new
    assert torch.equal(seq_g, seq_e)
    # log_softmax moves by at most twice the largest logit change; the score is a mean over the generated tokens
    assert float((sc_g - sc_e).abs().max()) <= 2 * budget, (float((sc_g - sc_e).abs().max()), budget)


def test_generate_with_cuda_graph_refusals():
    model = _model(256, 2, 2, 1)
    ids = torch.randint(0, 512, (1, 250), generator=torch.Generator().manual_seed(1)).cuda()
    with pytest.raises(ValueError, match="overflow"):
        model.generate(ids, max_new_tokens=20, use_cuda_graph=True)      # max_position_embeddings 256
    model.config.output_attentions = True
    with pytest.raises(ValueError, match="output_attentions"):
        model.generate(ids[:, :8], max_new_tokens=2, use_cuda_graph=True)


def test_vicuna_width_layer_step():
    """One layer at hidden 4096, 32 heads, 2048 cached rows: the graph step's layer output against `_forward_cached`'s (like-for-like:
    both against a float64 evaluation of the same layer on the same cache)."""
    from dreamllm_b200.decode import DecodeGraph
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    cfg = DreamLLMConfig(vocab_size=64, hidden_size=4096, intermediate_size=11008, num_hidden_layers=1, num_attention_heads=32,
                         max_position_embeddings=2304)
    torch.manual_seed(0)
    model = DreamLLMForCausalMLM(cfg).to(device="cuda", dtype=BF).eval()
    B, S = 2, 2048
    ids = torch.randint(0, 64, (B, S), generator=torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():
        out_e = model(input_ids=ids, use_cache=True, last_token_logits_only=True)
        out_g = model(input_ids=ids, use_cache=True, last_token_logits_only=True)
    nxt = out_e.logits[:, -1].argmax(-1)
    layer = model.model.layers[0]
    x = model.model.embed_tokens.weight.detach()[nxt][:, None].contiguous()
    with torch.no_grad():
        ye = layer(x, past_key_value=(out_e.past_key_values, 0), use_cache=True)[0][:, 0]
    # with one layer, the input of the final norm is the layer's output: read it there
    from dreamllm_b200 import ops
    captured, real = {}, ops.rmsnorm_fwd

    def spy(x2, w, eps, add=None, want_sum=True):
        if w is model.model.norm.weight:
            captured["y"] = x2.clone()
        return real(x2, w, eps, add=add, want_sum=want_sum)

    dg = DecodeGraph(model, out_g.past_key_values, B)
    dg.ids.copy_(nxt)
    ops.rmsnorm_fwd = spy
    try:
        dg.step()
    finally:
        ops.rmsnorm_fwd = real
    yg = captured["y"]
    # float64 reference of the same layer over the same cache rows
    sd = {k: v.detach().double().cpu() for k, v in layer.state_dict().items()}
    cache = out_e.past_key_values
    nh, d = 32, 128
    h = O.rmsnorm(x[:, 0].double().cpu(), sd["input_layernorm.weight"])
    qkv = h @ torch.cat([sd["self_attn.q_proj.weight"], sd["self_attn.k_proj.weight"], sd["self_attn.v_proj.weight"]]).T
    cos, sin = O.rope_tables(d, 4096, dtype=torch.float64)
    q = qkv[:, :4096].view(B, 1, nh, d).transpose(1, 2)
    k = qkv[:, 4096:8192].view(B, 1, nh, d).transpose(1, 2)
    q, k = O.apply_rope(q, k, cos, sin, torch.full((B, 1), S))
    Kc = torch.cat([cache.k[0][:, :S].double().cpu(), k.transpose(1, 2)], 1)
    Vc = torch.cat([cache.v[0][:, :S].double().cpu(), qkv[:, 8192:].view(B, 1, nh, d)], 1)
    att = torch.softmax(torch.einsum("bhd,blhd->bhl", q[:, :, 0], Kc) / math.sqrt(d), -1)
    ao = torch.einsum("bhl,blhd->bhd", att, Vc).reshape(B, 4096)
    xm = x[:, 0].double().cpu() + ao @ sd["self_attn.o_proj.weight"].T
    h2 = O.rmsnorm(xm, sd["post_attention_layernorm.weight"])
    gate, up = h2 @ sd["mlp.gate_proj.weight"].T, h2 @ sd["mlp.up_proj.weight"].T
    ref = xm + (torch.nn.functional.silu(gate) * up) @ sd["mlp.down_proj.weight"].T
    e_g = float((yg.double().cpu() - ref).abs().mean())
    e_e = float((ye.double().cpu() - ref).abs().mean())
    assert e_g <= 1.5 * e_e + 1e-6, (e_g, e_e)

"""Trainable CLIP vision tower (freeze_clip_vision_model=False and/or freeze_embedding_layers=False).

Kernels, one launch at a time, with the convention of test_tower_kernels_gpu.py: bf16 outputs within 1 ulp of the float64 reference
rounded once and at most 1 % of them differing at all; where a value cancels, the fp32 error of its terms (`atol`, derived beside each
assertion) may exceed an ulp of the result.  The tower against transformers' autograd (eager attention, same weights): every gradient
satisfies err(ours, fp32) <= 1.5 * err(transformers bf16, fp32), err = mean absolute difference.  Then the tower inside a
comprehension step, and one sharded AdamW step followed by the next forward.
"""
import math

import pytest
import torch

from oracle import tower_kernels_oracle as R

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64
EPS = 1e-5
SMALL = dict(hidden_size=256, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=4, image_size=56, patch_size=14)
VIT_L_336 = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16, image_size=336, patch_size=14)
ROWS = [(False, True), (False, False), (True, False)]        # (freeze_clip_vision_model, freeze_embedding_layers) with a trainable part


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _ops():
    from dreamllm_b200 import ops
    return ops


def _close_bf16(got, ref, atol=0.0, max_frac=1e-2, what=""):
    got = got.cpu()
    want = ref.to(torch.float32).to(BF)
    d = R.ulp_diff(got, want)
    err = (got.to(F64) - ref).abs()
    bad = (d > 1) & (err > atol + 2.0 ** -8 * ref.abs())
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements off by more than 1 ulp (worst {int(d.max())} ulp); "
                             f"first at flat index {i}: got {float(got.flatten()[i])}, reference {float(ref.flatten()[i])}")
    frac = float((d > 0).double().mean())
    assert frac <= max_frac, f"{what}: {frac:.4f} of the elements differ from the reference rounding (at most {max_frac} allowed)"


# ------------------------------------------------------------------------------------------------ LayerNorm affine backward
@pytest.mark.parametrize("T", [1, 577, 16 * 577])
# the three warp variants (<= 64, <= 128, <= 192 vectors per row); 1032 (129 vectors) leaves idle lanes in the warp kernel and a
# partly filled last 32-vector CTA in the weight pass
@pytest.mark.parametrize("H", [256, 1024, 1032, 1536])
def test_layernorm_bwd_affine_vs_float64(H, T):
    ops = _ops()
    x = (torch.randn(T, H, generator=_g(1), dtype=F64) * 2 + torch.randn(T, 1, generator=_g(2), dtype=F64)).to(BF)
    w = (1 + 0.3 * torch.randn(H, generator=_g(3))).to(BF)
    b = (0.3 * torch.randn(H, generator=_g(4))).to(BF)
    dy = torch.randn(T, H, generator=_g(5)).to(BF)
    dres = torch.randn(T, H, generator=_g(6)).to(BF)
    xd, wd, bd, dyd, rd = x.cuda(), w.cuda(), b.cuda(), dy.cuda(), dres.cuda()
    dx, dg, db = ops.layernorm_bwd_affine(dyd, xd, wd, EPS, dres=rd)
    assert torch.equal(dx, ops.layernorm_bwd(dyd, xd, wd, EPS, dres=rd)), "dx differs from layernorm_bwd"
    dx2, dg2, db2 = ops.layernorm_bwd_affine(dyd, xd, wd, EPS, dres=rd)
    assert torch.equal(dx, dx2) and torch.equal(dg, dg2) and torch.equal(db, db2), "two runs differ"
    x64, dy64 = x.to(F64), dy.to(F64)
    mean = x64.mean(1, keepdim=True)
    xhat = (x64 - mean) / torch.sqrt(((x64 - mean) ** 2).mean(1, keepdim=True) + EPS)
    t = dy64 * xhat
    # fp32: each term passes through at most ceil(T / 64 / 8) row adds, 8 group adds and 64 split adds, each with relative error
    # 2^-24 of the running sum (bounded by the sum of |terms|); xhat's mean / rstd contribute a few more 2^-24 of each term
    n_add = math.ceil(T / 64 / 8) + 8 + 64 + 4
    _close_bf16(dg, t.sum(0), atol=n_add * 2.0 ** -24 * t.abs().sum(0), what=f"dgamma H={H} T={T}")
    _close_bf16(db, dy64.sum(0), atol=n_add * 2.0 ** -24 * dy64.abs().sum(0), what=f"dbeta H={H} T={T}")
    # writing into caller buffers (gradient-bucket slices) gives the same bits
    og, ob = torch.empty_like(wd), torch.empty_like(wd)
    ops.layernorm_bwd_affine(dyd, xd, wd, EPS, dres=rd, dgamma=og, dbeta=ob)
    assert torch.equal(og, dg) and torch.equal(ob, db)


# ------------------------------------------------------------------------------------------------ quick-GELU
def _qg_inputs(n, seed):
    x = torch.randn(n, generator=_g(seed), dtype=F64) * 3
    x[: n // 4] = (torch.rand(n // 4, generator=_g(seed + 1), dtype=F64) * 2 - 1) * 40        # |x| up to 40: the saturated tails
    return x.to(BF)


def test_quick_gelu_fwd_bwd_vs_float64():
    ops = _ops()
    n = 1 << 20
    x = _qg_inputs(n, 10)
    dy = torch.randn(n, generator=_g(12)).to(BF)
    assert float(x.float().abs().max()) > 30
    y = ops.quick_gelu(x.cuda())
    x64, dy64 = x.to(F64), dy.to(F64)
    s = torch.sigmoid(1.702 * x64)
    # forward: exp and the divide carry a few 2^-24 relative, and the argument 1.702 x (|.| <= 68) is rounded to fp32, which moves
    # exp by up to 68 * 2^-24 relative: far below half a bf16 ulp, so only results at a rounding midpoint may land one ulp off
    _close_bf16(y, x64 * s, what="quick_gelu")
    # the fused GEMM epilogue applies the same formula: a bias-free identity GEMM through it gives the same bits
    eye = torch.eye(64, dtype=BF, device="cuda")
    xm = x[: 64 * 64].view(64, 64).cuda()
    assert torch.equal(ops.linear(xm, eye, act=ops.ACT_QUICK_GELU), y[: 64 * 64].view(64, 64))
    dx = ops.quick_gelu_bwd(dy.cuda(), x.cuda())
    t1, t2 = s, 1.702 * x64 * s * (1 - s)
    # backward: s + 1.702 x s (1 - s) cancels near x = -1.13; each term carries the relative error of s (<= 2^-16, as above) plus a
    # few fp32 roundings, so the absolute error is bounded by 2^-16 * |dy| * (|t1| + |t2|)
    _close_bf16(dx, dy64 * (t1 + t2), atol=2.0 ** -16 * dy64.abs() * (t1.abs() + t2.abs()), what="quick_gelu_bwd")


def test_quick_gelu_refuses_misaligned_pointers():
    ops = _ops()
    buf = torch.zeros(80, dtype=BF, device="cuda")
    with pytest.raises(RuntimeError, match="align"):
        ops.quick_gelu(buf[1:65])
    with pytest.raises(RuntimeError, match="align"):
        ops.quick_gelu_bwd(buf[1:65], buf[8:72])
    with pytest.raises(RuntimeError, match="align"):
        ops.layernorm_bwd_affine(buf[1:65].view(1, 64), buf[8:72].view(1, 64), buf[8:72], EPS)


def test_layernorm_bwd_affine_refuses_bad_arguments_before_launch():
    """Shape, workspace and pointer checks of the C entry, on real allocations sized for the call."""
    from dreamllm_b200._lib import lib
    L = lib()
    T, H = 577, 1024
    ws_bytes = L.dllm_layernorm_bwd_affine_workspace_bytes(T, H)
    t = torch.zeros(T, H + 8, dtype=BF, device="cuda")
    w = torch.zeros(2 * H, dtype=BF, device="cuda")
    ws = torch.zeros(ws_bytes + 64, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    P, Wp, WS = t.data_ptr(), w.data_ptr(), ws.data_ptr()
    err = lambda rc: L.dllm_error_string(rc).decode()                                                   # noqa: E731
    good = [P, P, Wp, None, P, Wp, Wp + 2 * H, WS]
    for i in (0, 1, 2, 4, 7):          # dy, x, w, dx, workspace 2 bytes off (dgamma / dbeta are stored element by element: bf16 alignment)
        bad = list(good)
        bad[i] += 2
        assert err(L.dllm_layernorm_bwd_affine(*bad, ws_bytes, T, H, EPS, st)) == err(-2), i
    shape = err(L.dllm_layernorm_bwd_affine(*good, ws_bytes - 4, T, H, EPS, st))                     # workspace too small
    assert shape == "invalid shape / size"
    assert err(L.dllm_layernorm_bwd_affine(*good, ws_bytes, T, H + 4, EPS, st)) == shape               # H % 8
    assert err(L.dllm_layernorm_bwd_affine(*good, ws_bytes, 4, 1544, EPS, st)) == shape                # wider than 192 vectors
    nul = list(good)
    nul[5] = None                                                                                      # no dgamma
    assert err(L.dllm_layernorm_bwd_affine(*nul, ws_bytes, T, H, EPS, st)) == shape
    assert err(L.dllm_quick_gelu(P, P, 12, st)) == shape                                              # n % 8
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ tower vs transformers
def _hf_clip(cfg_kw, dtype=torch.float32):
    from transformers import CLIPVisionConfig, CLIPVisionModel
    torch.manual_seed(0)
    cfg = CLIPVisionConfig(**cfg_kw)
    try:
        cfg._attn_implementation = "eager"
    except Exception:
        pass
    m = CLIPVisionModel(cfg)
    for p in m.parameters():          # non-trivial LN / bias values
        if p.dim() == 1:
            p.data.add_(0.05 * torch.randn_like(p))
    return m.to(dtype)


def _reference_flags(m, freeze_tower, freeze_emb, select_layer):
    """The reference's requires_grad_ calls (omni/models/dreamllm/modeling_plugins.py:248-257), restated."""
    m.requires_grad_(not freeze_tower)
    if not freeze_tower:
        for i in range(select_layer + 1, 0):
            m.vision_model.encoder.layers[i].requires_grad_(False)
        m.vision_model.post_layernorm.requires_grad_(False)
    m.vision_model.embeddings.requires_grad_(not freeze_emb)


def _plugin(cfg_kw, freeze_tower, freeze_emb, sd, freeze_projector=False):
    from dreamllm_b200.modeling_plugins import CLIPVisionEmbedding
    clip = CLIPVisionEmbedding(dict(cfg_kw), embed_hidden_size=256, freeze_clip_vision_model=freeze_tower,
                               freeze_embedding_layers=freeze_emb, freeze_projector=freeze_projector)
    clip.clip_vision_model.load_state_dict(sd)
    return clip.to(device="cuda", dtype=BF)


def _hf_grads(m, img, R_, select_layer=-2):
    m.zero_grad(set_to_none=True)
    feats = m(img, output_hidden_states=True).hidden_states[select_layer][:, 1:]
    (feats.float() * R_).sum().backward()
    return {n: p.grad.detach().float().cpu() for n, p in m.named_parameters() if p.requires_grad}


def _our_grads(tower, img, R_, select_layer=-2):
    for p in tower.parameters():
        p.grad = None
    feats = tower.hidden_state(img, select_layer)[:, 1:]
    (feats.float() * R_).sum().backward()
    return {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in tower.named_parameters()}


def _check_tower_grads(cfg_kw, n_img, freeze_tower, freeze_emb):
    hf32 = _hf_clip(cfg_kw).cuda()
    sd = hf32.state_dict()
    hfbf = _hf_clip(cfg_kw, BF).cuda()
    hfbf.load_state_dict(sd)
    for m in (hf32, hfbf):
        _reference_flags(m, freeze_tower, freeze_emb, -2)
    clip = _plugin(cfg_kw, freeze_tower, freeze_emb, sd)
    tower = clip.clip_vision_model
    r = cfg_kw["image_size"]
    img = torch.randn(n_img, 3, r, r, generator=_g(21)).cuda()
    P = (r // cfg_kw["patch_size"]) ** 2
    R_ = torch.randn(n_img, P, cfg_kw["hidden_size"], generator=_g(22)).cuda()
    g32 = _hf_grads(hf32, img, R_)
    gbf = _hf_grads(hfbf, img.to(BF), R_)
    ours = _our_grads(tower, img.to(BF), R_)
    trainable = {n for n, p in tower.named_parameters() if p.requires_grad}
    assert trainable == set(g32), "the plugin's trainable set is the reference's"
    for n, g in ours.items():
        if n not in trainable:
            assert g is None, f"{n} is frozen but got a gradient"
    layers_run = cfg_kw["num_hidden_layers"] - 1                     # select_layer -2: the last layer is never computed
    ratios, bad = [], []
    for n in sorted(trainable):
        if n.startswith(f"vision_model.encoder.layers.{layers_run}.") or n.startswith("vision_model.post_layernorm"):
            continue                                                  # frozen by the select_layer rule, never computed here
        got = ours[n]
        assert got is not None, f"{n} requires grad but got none"
        if n.endswith("k_proj.bias"):
            assert not bool(got.any()), f"{n}: the gradient of a key bias is exactly zero"
        e_o = float((got.float().cpu() - g32[n]).abs().mean())
        e_r = float((gbf[n] - g32[n]).abs().mean())
        ratios.append((round(e_o / max(e_r, 1e-30), 3), n))
        if not e_o <= 1.5 * e_r:
            bad.append(f"{n}: err {e_o:.3e} > 1.5 x transformers bf16 err {e_r:.3e}")
    print("worst err(ours) / err(transformers bf16):", sorted(ratios)[-5:])
    assert not bad, "\n".join(bad)
    again = _our_grads(tower, img.to(BF), R_)
    for n, g in ours.items():
        assert (g is None and again[n] is None) or torch.equal(g, again[n]), f"{n}: two backwards differ"


@pytest.mark.parametrize("freeze_tower,freeze_emb", ROWS)
def test_small_tower_grads_vs_transformers(freeze_tower, freeze_emb):
    _check_tower_grads(SMALL, 3, freeze_tower, freeze_emb)


@pytest.mark.parametrize("freeze_tower,freeze_emb", ROWS[:2])
def test_vit_l_336_grads_vs_transformers(freeze_tower, freeze_emb):
    _check_tower_grads(VIT_L_336, 2, freeze_tower, freeze_emb)


# frozen forward launches (ops.LAUNCHES): patchify, patch GEMM + its split-K reduce, assemble, pre_layrnorm = 5; per computed layer
# LN1, q|k|v GEMM, attention, out_proj, LN2, fc1, fc2 + its split-K reduce = 8, and at ViT-L/14-336 out_proj runs split-K too (9)
@pytest.mark.parametrize("cfg_kw,n_img,launches", [(SMALL, 3, 5 + 2 * 8), (VIT_L_336, 2, 5 + 23 * 9)])
def test_frozen_tower_vs_transformers(cfg_kw, n_img, launches):
    """The plugin's default flags: the no_grad forward with the fused quick-GELU epilogue, the row-fused q|k|v weight and the cached
    padded patch weight, against transformers with the same weights (like-for-like bound of test_clip_splice_gpu.py)."""
    from dreamllm_b200 import ops
    hf = _hf_clip(cfg_kw)
    hfb = _hf_clip(cfg_kw, BF)
    hfb.load_state_dict(hf.state_dict())
    clip = _plugin(cfg_kw, True, True, hf.state_dict())
    tower = clip.clip_vision_model
    assert not any(p.requires_grad for p in tower.parameters())
    r = cfg_kw["image_size"]
    img = torch.randn(n_img, 3, r, r, generator=_g(23))
    for sel in (-2, 0):
        with torch.no_grad():
            ref32 = hf(img, output_hidden_states=True).hidden_states[sel]
            refbf = hfb(img.to(BF), output_hidden_states=True).hidden_states[sel].float()
        ops.LAUNCHES.reset()
        got = tower.hidden_state(img.cuda().to(BF), sel)
        if sel == -2:
            assert ops.LAUNCHES.count == launches
        assert got.grad_fn is None and not got.requires_grad
        got = got.float().cpu()
        e_o, e_r = float((got - ref32).abs().mean()), float((refbf - ref32).abs().mean())
        assert e_o <= 1.3 * e_r + 1e-3 * float(ref32.abs().mean()), (sel, e_o, e_r)


# ------------------------------------------------------------------------------------------------ inside a comprehension step
@pytest.mark.parametrize("freeze_projector", [False, True])
def test_comprehension_step_tower_grads_equal_tower_backward(freeze_projector):
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    from dreamllm_b200.modeling_plugins import CLIPVisionEmbedding, DreamEmbedding
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=32008, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2)
    m = DreamLLMForCausalMLM(cfg)
    clip = CLIPVisionEmbedding(dict(SMALL), embed_hidden_size=256, freeze_clip_vision_model=False, freeze_embedding_layers=False,
                               freeze_projector=freeze_projector)
    dream = DreamEmbedding(num_dream_queries=8, embed_hidden_size=256)
    m.model.attach_plugins(clip, dream, image_start_id=32003, dream_start_id=32006)
    m = m.to(device="cuda", dtype=BF)
    P = clip.embed_len
    ids = torch.full((2, 64), 32000)
    ids[0, :P + 6] = torch.tensor([1, 32003] + [32002] * P + [32004, 5, 6, 2])
    ids[1, :P + 5] = torch.tensor([1, 32003] + [32002] * P + [32004, 7, 2])
    labels = ids.clone()
    labels[ids >= 32000] = -100
    imgs = torch.randn(2, 3, 56, 56, generator=_g(24)).to(BF).cuda()
    captured = []
    proj_fwd = clip.projector.forward

    def spy(features):
        if features.requires_grad:
            features.register_hook(lambda g: captured.append(g.detach().clone()))
        return proj_fwd(features)

    clip.projector.forward = spy
    out = m(input_ids=ids.cuda(), images=imgs, attention_mask=(ids != 32000).long().cuda(), labels=labels.cuda(), input_ids_cpu=ids)
    out.loss.backward()
    tower = clip.clip_vision_model
    got = {n: p.grad for n, p in tower.named_parameters()}
    if freeze_projector:
        # the reference's frozen projector runs under set_grad_enabled(False) (mlp_projector.py), so no gradient reaches the tower
        assert not captured and all(g is None for g in got.values())
        return
    assert len(captured) == 1 and torch.isfinite(out.loss)
    got = {n: g.clone() for n, g in got.items() if g is not None}
    assert got and set(got) == {n for n, p in tower.named_parameters() if p.requires_grad and not n.startswith(
        ("vision_model.encoder.layers.2.", "vision_model.post_layernorm"))}
    for p in tower.parameters():
        p.grad = None
    tower.hidden_state(imgs, clip.select_layer)[:, 1:].backward(captured[0])
    for n, g in got.items():
        assert torch.equal(g, tower.get_parameter(n).grad), f"{n}: the step's tower gradient is not the tower backward of its input"


# ------------------------------------------------------------------------------------------------ sharded AdamW
def test_sharded_adamw_step_then_forward(tmp_path, monkeypatch):
    import torch.distributed as dist

    from dreamllm_b200 import ops
    from dreamllm_b200.zero import ShardedAdamW
    own_pg = not dist.is_initialized()
    if own_pg:
        dist.init_process_group("gloo", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0, world_size=1)
    try:
        hf = _hf_clip(SMALL)
        clip = _plugin(SMALL, False, False, hf.state_dict())
        tower = clip.clip_vision_model
        opt = ShardedAdamW([p for p in tower.parameters() if p.requires_grad], lr=1e-2, weight_decay=0.01).attach(tower)
        img = torch.randn(3, 3, 56, 56, generator=_g(25)).cuda().to(BF)
        R_ = torch.randn(3, 16, 256, generator=_g(26)).cuda()
        outs = []
        wgrad = ops.linear_wgrad
        monkeypatch.setattr(ops, "linear_wgrad", lambda dy, x, out=None, **kw: outs.append(out) or wgrad(dy, x, out=out, **kw))
        for step in range(2):
            outs.clear()
            (tower.hidden_state(img, -2)[:, 1:].float() * R_).sum().backward()
            ptrs = {o.data_ptr() for o in outs if o is not None}
            for li in range(2):
                lyr = tower.vision_model.encoder.layers[li]
                for p in (lyr.self_attn.q_proj.weight, lyr.self_attn.k_proj.weight, lyr.self_attn.v_proj.weight,
                          lyr.self_attn.out_proj.weight, lyr.mlp.fc1.weight, lyr.mlp.fc2.weight):
                    assert opt._bucket_of[p].gviews[p].data_ptr() in ptrs, "a weight gradient was not written into its bucket"
            opt.step(defer_gather=True)                  # raises if a parameter left its bucket
            opt.zero_grad()
        # one forward with the flags off: the frozen path must leave the optimizer's parameters in their buckets and must not serve the
        # padded patch weight cached before the step
        trainable = [p for p in tower.parameters() if p.requires_grad]
        tower.requires_grad_(False)
        frozen_feats = tower.hidden_state(img, -2).float().cpu()
        for p in trainable:
            p.requires_grad_(True)
        assert all(p.data_ptr() == opt._bucket_of[p].pviews[p].data_ptr() for p in trainable)
        # the next forward sees the updated weights (a stale padded patch weight would not)
        sd = {k: v.float().cpu() for k, v in tower.state_dict().items()}
        hf.load_state_dict(sd)
        hfb = _hf_clip(SMALL, BF)
        hfb.load_state_dict(sd)
        with torch.no_grad():
            ref32 = hf(img.float().cpu(), output_hidden_states=True).hidden_states[-2]
            refbf = hfb(img.cpu(), output_hidden_states=True).hidden_states[-2].float()
            got = tower.hidden_state(img, -2).float().cpu()
        e_r = float((refbf - ref32).abs().mean())
        for feats in (got, frozen_feats):
            e_o = float((feats - ref32).abs().mean())
            assert e_o <= 1.3 * e_r + 1e-3 * float(ref32.abs().mean()), (e_o, e_r)
    finally:
        if own_pg:
            dist.destroy_process_group()

"""SDXL head on the GPU: UNet-XL forward against the fp32 from-spec oracle (oracle/unet_xl_oracle.py), the dgrad-only backward into the
cross-attention conditioning and the pooled text_embeds against oracle autograd, the new kernels, the XL head's loss and gradients, the
graph-captured CFG loop and a stage-1 creation step through DreamLLMForCausalMLM.  Criterion as test_unet_gpu.py: the native bf16 path's
error against the fp32 oracle stays within the error of the oracle's own bf16 run."""
import pytest
import torch

from oracle import unet_oracle as UO
from oracle import unet_xl_oracle as XO

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
CT = 256          # text_embeds width of the small config (= its time-embedding width, as 1280 is SDXL's)
SMALL_XL = dict(block_out_channels=(64, 128, 256), attention_head_dim=(1, 2, 4), cross_attention_dim=128, down_attn=(False, True, True),
                up_attn=(True, True, False), transformer_layers_per_block=(1, 2, 3), addition_embed_type="text_time",
                addition_time_embed_dim=256, projection_class_embeddings_input_dim=CT + 6 * 256)
SMALL_VAE = dict(block_out_channels=(64, 128, 128, 128))
IDS = [[1024., 1024., 0., 0., 1024., 1024.], [768., 1344., 16., 32., 1024., 1024.], [896., 1152., 64., 0., 1024., 1024.]]


def _rel(a, ref):
    return float((a - ref).abs().mean() / ref.abs().mean())


def _pair(cfg, seed=0):
    from dreamllm_b200.unet import UNet2DConditionModel
    torch.manual_seed(seed)
    ref = XO.UNet2DConditionModel(cfg).eval()
    for n, p in ref.named_parameters():
        if p.dim() == 1 and "norm" in n and n.endswith("weight"):
            p.data.add_(0.1 * torch.randn_like(p))
        elif p.dim() == 1:
            p.data.add_(0.02 * torch.randn_like(p))
    ours = UNet2DConditionModel(cfg)
    assert [(k, tuple(v.shape)) for k, v in ours.state_dict().items()] == [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    ours.load_state_dict(ref.state_dict())
    return ref, ours.to(device="cuda", dtype=BF)


def _bf16_ref(ref, cfg):
    r = XO.UNet2DConditionModel(cfg).eval()
    r.load_state_dict(ref.state_dict())
    return r.to(BF)


def _ids(B):
    return torch.tensor(IDS[:B] + IDS[:max(0, B - len(IDS))])


@pytest.mark.parametrize("B,HW,Q", [(2, 16, 7), (3, 32, 77)])
def test_unet_xl_forward_small_vs_oracle(B, HW, Q):
    ref, ours = _pair(SMALL_XL)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 4, HW, HW, generator=g)
    c = torch.randn(B, Q, 128, generator=g)
    text = torch.randn(B, CT, generator=g)
    ids = _ids(B)
    t = 481
    with torch.no_grad():
        want = ref(x, torch.tensor(t), c, dict(text_embeds=text, time_ids=ids))
        wantb = _bf16_ref(ref, SMALL_XL)(x.to(BF), torch.tensor(t), c.to(BF), dict(text_embeds=text.to(BF), time_ids=ids.to(BF))).float()
    got = ours(x.cuda(), t, c.cuda(), dict(text_embeds=text.cuda().to(BF), time_ids=ids.cuda())).cpu()
    e_o, e_r = _rel(got, want), _rel(wantb, want)
    print(f"rel err ours {e_o:.4f} ref-bf16 {e_r:.4f}")
    assert e_o <= 1.5 * e_r + 5e-3, (e_o, e_r)
    # the addition embedding carries signal: other time ids give another prediction
    other = ours(x.cuda(), t, c.cuda(), dict(text_embeds=text.cuda().to(BF), time_ids=ids.cuda() * 0.5)).cpu()
    assert not torch.equal(other, got)


def test_unet_xl_forward_full_width():
    """real SDXL widths (320/640/1280, heads 5/10/20, depth 1/2/10, ctx 2048) on 32x32 latents, B 1, Q 196; fp32 oracle on the host."""
    from dreamllm_b200.unet import SDXL
    ref, ours = _pair(SDXL, seed=3)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 4, 32, 32, generator=g)
    c = torch.randn(1, 196, 2048, generator=g)
    text = torch.randn(1, 1280, generator=g)
    ids = _ids(1)
    with torch.no_grad():
        want = ref(x, torch.tensor(961), c, dict(text_embeds=text, time_ids=ids))
    del ref
    got = ours(x.cuda(), 961, c.cuda().to(BF), dict(text_embeds=text.cuda().to(BF), time_ids=ids.cuda())).cpu()
    e = _rel(got, want)
    print(f"full-width rel err {e:.4f}")
    assert e < 4e-2, e


@pytest.mark.parametrize("zero_cross_out", [False, True], ids=["both", "pooled-only"])
def test_unet_xl_cond_and_text_gradients_vs_oracle_autograd(zero_cross_out):
    """d(loss)/d(cond) and d(loss)/d(text_embeds) through the frozen UNet-XL.  pooled-only: every cross-attention output projection is
    zeroed (in both models), so the loss reaches the conditioning only through the time embedding: dcond is exactly 0 and dtext carries
    the whole gradient."""
    from dreamllm_b200 import ops
    ref, ours = _pair(SMALL_XL, seed=11)
    if zero_cross_out:
        for m in (ref, ours):
            for n, p in m.named_parameters():
                if ".attn2.to_out.0." in n:
                    p.data.zero_()
    B, HW, Q = 2, 16, 7
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(B, 4, HW, HW, generator=g)
    noise = torch.randn(B, 4, HW, HW, generator=g)
    t = torch.tensor([113, 877])
    cond = torch.randn(B, Q, 128, generator=g)
    text = torch.randn(B, CT, generator=g)
    ids = _ids(B)
    ac = UO.alphas_cumprod()
    noisy = UO.add_noise(x0, noise, t, ac)
    c32, t32 = cond.clone().requires_grad_(True), text.clone().requires_grad_(True)
    loss = torch.nn.functional.mse_loss(ref(noisy, t, c32, dict(text_embeds=t32, time_ids=ids)), noise)
    loss.backward()
    refb = _bf16_ref(ref, SMALL_XL)
    cb, tb = cond.to(BF).requires_grad_(True), text.to(BF).requires_grad_(True)
    torch.nn.functional.mse_loss(refb(noisy.to(BF), t, cb, dict(text_embeds=tb, time_ids=ids.to(BF))).float(), noise).backward()
    noisy_c = ops.add_noise(x0.cuda(), noise.cuda(), t.int().cuda(), ac.cuda())
    eps, tape = ours.forward_train(noisy_c, t.int().cuda(), cond.cuda().to(BF), (text.cuda().to(BF), ids.cuda()))
    l, deps = ops.mse_fwd_bwd(eps, noise.cuda())
    dcond, dtext = ours.backward_cond(deps, tape)
    assert abs(float(l) - float(loss)) < 3e-2 * float(loss)
    e_t, e_tr = _rel(dtext.cpu().float(), t32.grad), _rel(tb.grad.float(), t32.grad)
    print(f"dtext rel err ours {e_t:.4f} ref-bf16 {e_tr:.4f}")
    assert e_t <= 1.5 * e_tr + 2e-2, (e_t, e_tr)
    if zero_cross_out:
        assert float(dcond.abs().max()) == 0.0 and float(c32.grad.abs().max()) == 0.0
    else:
        e_c, e_cr = _rel(dcond.cpu().float(), c32.grad), _rel(cb.grad.float(), c32.grad)
        print(f"dcond rel err ours {e_c:.4f} ref-bf16 {e_cr:.4f}")
        assert e_c <= 1.5 * e_cr + 2e-2, (e_c, e_cr)
    # the tape-recording forward is the inference forward, bit for bit, where both take one shared timestep
    t1 = torch.full((B,), 113, dtype=torch.int32, device="cuda")
    eps1, _ = ours.forward_train(noisy_c, t1, cond.cuda().to(BF), (text.cuda().to(BF), ids.cuda()))
    assert torch.equal(eps1, ours(noisy_c, 113, cond.cuda().to(BF), dict(text_embeds=text.cuda().to(BF), time_ids=ids.cuda())))
    # without added_cond an XL UNet is refused
    with pytest.raises(ValueError, match="text_embeds"):
        ours.forward_train(noisy_c, t1, cond.cuda().to(BF))


@pytest.mark.parametrize("N,HW,C", [(1, 16384, 320), (2, 4096, 640), (4, 196, 4096), (3, 77, 1280), (2, 5, 24)])
def test_channel_sum_vs_float64_and_deterministic(N, HW, C):
    from dreamllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(N * HW + C)
    x = torch.randn(N, HW, C, device="cuda", generator=g).to(BF)
    want = x.double().sum(1)
    got = ops.channel_sum_nhwc(x)
    assert got.dtype == torch.float32 and got.shape == (N, C)
    assert float((got.double() - want).abs().max()) <= 1e-5 * HW ** 0.5 * 4 + 1e-4
    assert torch.equal(got, ops.channel_sum_nhwc(x))
    # column slice of a wider buffer, bf16, scaled: the mean over the middle axis, rounded once
    wide = torch.full((N, C + 40), 7.0, device="cuda", dtype=BF)
    ops.channel_sum_nhwc(x, out=wide[:, 16:16 + C], scale=1.0 / HW)
    assert float((wide[:, 16:16 + C].double() - want / HW).abs().max()) <= 2 ** -8 * float((want / HW).abs().max())
    assert bool((wide[:, :16] == 7).all()) and bool((wide[:, 16 + C:] == 7).all())
    m = ops.mean_rows(x)
    assert torch.equal(m, wide[:, 16:16 + C])
    ref = x.mean(1)                                               # torch.mean of bf16: fp32 accumulate, one rounding
    assert float((m.float() - ref.float()).abs().max()) <= 2 ** -7 * float(ref.float().abs().max())


def test_small_kernels_vs_formulas():
    from dreamllm_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.randn(4, 1280, device="cuda", generator=g) * 3).to(BF)
    dy = torch.randn(4, 1280, device="cuda", generator=g).to(BF)
    xf = x.float()
    assert float((ops.silu(x).float() - torch.nn.functional.silu(xf)).abs().max()) <= 2 ** -7 * float(xf.abs().max())
    s = torch.sigmoid(xf)
    want = dy.float() * s * (1 + xf * (1 - s))
    assert float((ops.silu_bwd(dy, x).float() - want).abs().max()) <= 2 ** -7 * float(want.abs().max())
    # the separate SiLU rounds as the GEMM's fused one
    w = (torch.randn(1280, 1280, device="cuda", generator=g) * 0.03).to(BF)
    assert torch.equal(ops.linear(x, w, act=ops.ACT_SILU), ops.silu(ops.linear(x, w)))
    b = ops.broadcast_rows(dy, 5, 0.25)
    assert b.shape == (4, 5, 1280) and torch.equal(b, (dy.float() * 0.25).to(BF)[:, None].expand(4, 5, 1280))
    ids = torch.tensor(IDS, device="cuda")
    out = torch.zeros(3, 1280 + 6 * 256 + 8, device="cuda", dtype=BF)
    ops.time_ids_embedding(ids, out[:, 1280:1280 + 6 * 256])
    te = UO.timestep_embedding(ids.cpu().flatten(), 256).reshape(3, -1)
    assert float((out[:, 1280:1280 + 1536].cpu().float() - te).abs().max()) <= 2 ** -8
    assert bool((out[:, :1280] == 0).all()) and bool((out[:, -8:] == 0).all())


def _small_xl_head(seed):
    from dreamllm_b200.modeling_plugins import StableDiffusionXLHead
    torch.manual_seed(seed)
    cfg = dict(SMALL_XL)
    cfg["vae"] = SMALL_VAE
    head = StableDiffusionXLHead(cfg, embed_hidden_size=256, global_condition_hidden_size=CT)
    ref = XO.UNet2DConditionModel(SMALL_XL).eval()
    ref.load_state_dict(head.unet.state_dict())
    wp = head.projector.projector.weight.detach().clone()
    wg, bg = head.global_projector.projector.weight.detach().clone(), head.global_projector.projector.bias.detach().clone()
    bg.normal_(0, 0.1)
    head.global_projector.projector.bias.data.copy_(bg)
    return head.to(device="cuda", dtype=BF), ref, wp, wg, bg


def test_xl_head_loss_and_grads_vs_oracle():
    """reference dreamllm_sdxl/modeling_plugins.py:151-236 with the projector, the global projector and the mean over dream queries."""
    head, ref, wp, wg, bg = _small_xl_head(2)
    assert head.vae.cfg["scaling_factor"] == 0.13025 and head.save_model_name == "stable_diffusion_xl_head"
    g = torch.Generator().manual_seed(3)
    Nd, Q = 2, 8
    lat = torch.randn(Nd, 4, 16, 16, generator=g) * 0.5
    enc = torch.randn(Nd, Q, 256, generator=g)
    noise = torch.randn(Nd, 4, 16, 16, generator=g)
    t = torch.tensor([17, 803])
    ids = _ids(Nd)
    e32 = enc.clone().requires_grad_(True)
    wp32, wg32, bg32 = wp.clone().requires_grad_(True), wg.clone().requires_grad_(True), bg.clone().requires_grad_(True)
    text = torch.nn.functional.linear(e32.mean(1), wg32, bg32)
    noisy = UO.add_noise(lat, noise, t, UO.alphas_cumprod())
    pred = ref(noisy, t, torch.nn.functional.linear(e32, wp32), dict(text_embeds=text, time_ids=ids))
    want = torch.nn.functional.mse_loss(pred, noise)
    want.backward()
    ec = enc.cuda().to(BF).requires_grad_(True)
    loss = head(None, ec, None, ids.cuda(), latents=lat.cuda(), noise=noise.cuda(), timesteps=t.cuda())
    loss.backward()
    print(f"xl head loss {float(loss):.5f} want {float(want):.5f}")
    assert abs(float(loss) - float(want)) < 5e-2 * float(want)
    assert _rel(ec.grad.cpu().float(), e32.grad) < 0.15
    assert _rel(head.projector.projector.weight.grad.cpu().float(), wp32.grad) < 0.15
    assert _rel(head.global_projector.projector.weight.grad.cpu().float(), wg32.grad) < 0.15
    assert _rel(head.global_projector.projector.bias.grad.cpu().float(), bg32.grad) < 0.15
    assert all(p.grad is None for p in head.unet.parameters())
    with pytest.raises(ValueError, match="add_time_ids"):
        head(None, ec, latents=lat.cuda(), noise=noise.cuda(), timesteps=t.cuda())


def test_xl_pipeline_graph_equals_eager_with_cfg():
    head, ref, wp, wg, bg = _small_xl_head(4)
    g = torch.Generator().manual_seed(9)
    B, Q, N = 2, 8, 4
    pos = torch.randn(B, Q, 256, generator=g).cuda().to(BF)
    neg = torch.randn(B, Q, 256, generator=g).cuda().to(BF)
    lat0 = torch.randn(B, 4, 16, 16, generator=g).cuda()
    kw = dict(height=128, width=128, num_inference_steps=N, guidance_scale=5.0, latents=lat0, prompt_embeds=pos,
              negative_prompt_embeds=neg, scheduler="ddim")
    a = head.pipeline(**kw)
    b = head.pipeline(use_cuda_graph=False, **kw)
    assert torch.equal(a, b) and torch.isfinite(a).all()
    # the oracle loop: diffusers' SDXL pipeline order (uncond first), default time ids (1024, 1024, 0, 0, 1024, 1024)
    ids = torch.tensor([[1024., 1024., 0., 0., 1024., 1024.]] * (2 * B))
    encs = torch.cat([neg, pos]).float().cpu()
    cond = torch.nn.functional.linear(encs, wp)
    text = torch.nn.functional.linear(encs.mean(1), wg, bg)
    ac, ts = UO.alphas_cumprod(), UO.set_timesteps(N)
    lat = lat0.cpu()
    with torch.no_grad():
        for tt in ts.tolist():
            e = ref(torch.cat([lat] * 2), torch.tensor(tt), cond, dict(text_embeds=text, time_ids=ids))
            eu, ec = e.chunk(2)
            lat = UO.ddim_step(lat, UO.cfg_combine(eu, ec, 5.0), tt, 1000 // N, ac)
    rel = _rel(a.cpu(), lat)
    print(f"xl cfg loop rel err {rel:.4f}")
    assert rel < 5e-2, rel
    # other micro-conditioning changes the sample
    c = head.pipeline(original_size=(512, 512), **kw)
    assert not torch.equal(c, a)


def test_xl_creation_step_end_to_end():
    """stage-1 creation with the XL head: add_time_ids from the batch, gradients reach the dream queries through both conditioning
    paths; add_time_ids missing in training, or given to a model whose head is SD-2.1, is refused."""
    from dreamllm_b200.modeling_dreamllm import DreamLLMConfig, DreamLLMForCausalMLM
    from dreamllm_b200.modeling_plugins import DreamEmbedding, StableDiffusionXLHead
    torch.manual_seed(0)
    cfg = DreamLLMConfig(vocab_size=32008, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2)
    m = DreamLLMForCausalMLM(cfg)
    Q = 8
    dream = DreamEmbedding(num_dream_queries=Q, embed_hidden_size=256)
    sdc = dict(SMALL_XL)
    sdc["vae"] = SMALL_VAE
    m.stable_diffusion_head = StableDiffusionXLHead(sdc, embed_hidden_size=256, global_condition_hidden_size=CT)
    m.model.attach_plugins(None, dream, image_start_id=32003, dream_start_id=32006)
    m = m.to(device="cuda", dtype=BF)
    for p in m.parameters():
        p.requires_grad_(False)
    dream.dream_queries.requires_grad_(True)
    m.stable_diffusion_head.projector.requires_grad_(True)
    m.stable_diffusion_head.global_projector.requires_grad_(True)
    m.train()
    B, S = 2, 32
    ids = torch.full((B, S), 32000)
    for b in range(B):
        row = [1, 11 + b, 12, 32006] + [32002] * Q + [32007, 2]
        ids[b, :len(row)] = torch.tensor(row)
    labels = torch.full((B, S), -100)
    am = (ids != 32000).long()
    imgs = (torch.rand(B, 3, 128, 128) * 2 - 1).to(BF)
    kw = dict(input_ids=ids.cuda(), images_dm=imgs.cuda(), attention_mask=am.cuda(), labels=labels.cuda(), input_ids_cpu=ids)
    with pytest.raises(ValueError, match="add_time_ids"):
        m(**kw)
    out = m(add_time_ids=_ids(B).cuda(), **kw)
    out.loss.backward()
    assert torch.isfinite(out.loss) and float(out.additional_log_info["vm_loss"]) > 0
    gq = dream.dream_queries.grad
    assert gq is not None and torch.isfinite(gq.float()).all() and float(gq.float().abs().sum()) > 0
    assert m.stable_diffusion_head.global_projector.projector.weight.grad is not None
    assert m.model.layers[0].mlp.down_proj.weight.grad is None

"""Host-side checks of the flash-attention float64 restatements, probes and comparison (oracle/attn_oracle.py), no GPU:

* with rounding switched off the restatements are plain float64 softmax attention and its autograd, with GQA as `gqa_oracle.repeat_kv`;
* the probes' closed forms (counts and integer sums) equal the restatements on the probe inputs;
* the comparison tests/test_attn_float64_gpu.py applies rejects a kernel that is subtly wrong: faults a kernel could plausibly have
  (a mask boundary off by one, a dropped tile edge key, visible fill keys, the wrong kv head, a missed rescale, the wrong lse units, a
  backward kernel starting or stopping one tile or key off, a dropped GQA head, a packed tile's tail seen as keys) are injected into
  the restatement on the GPU test's own inputs, and each is rejected with 10x C_ACC / C_LSE (or 10x the probe tolerance) in at least
  one case of the table;
* an fp32 emulation of the kernels, rounding to bf16 where they do, passes the comparison: the bound is not tighter than fp32
  arithmetic allows.
"""
import pytest
import torch

from oracle import attn_oracle as R
from oracle import gqa_oracle as G

F64 = torch.float64
F32 = torch.float32


def _find(**kw):
    for c in R.CASES:
        if all(getattr(c, k) == v for k, v in kw.items()):
            return c
    raise LookupError(kw)


# small cases of the table, one per kind / branch family
SMALL = [
    _find(kind="self", S=129, d=64, causal=True, seqlens=None, nh=2, nkv=2, dist="normal"),
    _find(kind="self", S=65, d=128, causal=False, nh=2, nkv=2, dist="normal"),
    _find(kind="self", B=9, causal=True),
    _find(kind="self", nh=8, nkv=4),
    _find(kind="cross", S=64, Skv=77),
    _find(kind="cache", S=5, mask=True),
    _find(kind="cache", S=1, Skv=128, mask=False),
    _find(kind="packed", d=128, causal=True),
    _find(kind="packed", d=64, causal=False),
    _find(kind="self", S=384, causal=True, dist="rise"),
    _find(kind="self", S=257, scale=0.3),
]


def _plain(q, k, v, vis, qrow, scale):
    """Softmax attention in float64 with repeat_kv: (out [B, S, nh, d], lse [B, nh, S]); rows without a visible key give 0 / +inf."""
    nh = q.shape[2]
    rep = nh // k.shape[2]
    kk = G.repeat_kv(k.to(F64).permute(0, 2, 1, 3), rep)
    vv = G.repeat_kv(v.to(F64).permute(0, 2, 1, 3), rep)
    s = (q.to(F64).permute(0, 2, 1, 3) @ kk.transpose(-1, -2)) * scale
    s = s.masked_fill(~vis[:, None], -float("inf"))
    lse = torch.logsumexp(s, -1)
    ok = torch.isfinite(lse) & qrow[:, None]
    p = torch.where(ok[..., None], torch.exp(s - torch.where(ok, lse, 0.0)[..., None]), 0.0)
    return (p @ vv).permute(0, 2, 1, 3), torch.where(ok, lse, float("inf"))


# ------------------------------------------------------------------------------------------------ the restatements
@pytest.mark.parametrize("case", SMALL, ids=[c.id for c in SMALL])
def test_unrounded_restatement_is_softmax_attention_and_autograd(case):
    inp = R.make_inputs(case)
    for rows, q, k, v, vis, qrow in R.subproblems(case, inp):
        pre, lse, _ = R.fwd_ref(q, k, v, vis, qrow, case.scale_v, rnd=False)
        out, lse_p = _plain(q, k, v, vis, qrow, case.scale_v)
        assert torch.allclose(pre, out, rtol=1e-10, atol=1e-12)
        assert torch.equal(torch.isinf(lse), torch.isinf(lse_p))
        fin = torch.isfinite(lse_p)
        assert torch.allclose(lse[fin], lse_p[fin], rtol=1e-12, atol=1e-12)
        if not case.has_bwd:
            continue
        r = rows if rows is not None else slice(None)
        do = inp["dout"].reshape(*(1, case.S) if case.kind == "packed" else (case.B, case.S), case.nh, case.d)[:, r].to(F64)
        qa, ka, va = (t.to(F64).requires_grad_(True) for t in (q, k, v))
        o_a, _ = _plain(qa, ka, va, vis, qrow, case.scale_v)
        (o_a * do).sum().backward()
        (dq, dk, dv), _ = R.bwd_ref(q, k, v, out, lse_p, do, vis, vis, qrow, case.scale_v, rnd=False)
        for got, want in ((dq, qa.grad), (dk, ka.grad), (dv, va.grad)):
            assert torch.allclose(got, want, rtol=1e-9, atol=1e-11), float((got - want).abs().max())


def test_kv_head_map_is_repeat_kv():
    for nh, nkv in ((8, 8), (8, 4), (32, 8), (32, 1)):
        x = torch.arange(nkv, dtype=F64)[None, :, None, None].expand(1, nkv, 3, 2)
        assert torch.equal(G.repeat_kv(x, nh // nkv)[0, :, 0, 0].long(), R.kv_head_map(nh, nkv))
    assert not torch.equal(R.kv_head_map(8, 4, "gqa_mod"), R.kv_head_map(8, 4))


def test_tile_walk_rounds_p_at_the_running_max():
    """One row, two tiles: the second tile's larger key rescales the first tile's already-rounded weights (they are not re-rounded)."""
    q = torch.zeros(1, 1, 1, 64, dtype=torch.bfloat16)
    q[..., 0] = 1.0
    k = torch.zeros(1, 256, 1, 64, dtype=torch.bfloat16)
    k[0, 0, 0, 0], k[0, 128, 0, 0] = 0.3, 1.7
    v = torch.randn(1, 256, 1, 64, generator=torch.Generator().manual_seed(3)).to(torch.bfloat16)
    vis, qrow = R.visibility(1, 1, 256, False)
    pre, lse, _ = R.fwd_ref(q, k, v, vis, qrow, 1.0)
    c = R.fl32(R.LOG2E)
    s = k[0, :, 0, 0].to(F64) * c
    p1 = R.bf16r(torch.exp2(s[:128] - s[:128].max()))
    m2 = s.max()
    p2 = R.bf16r(torch.exp2(s[128:] - m2))
    a = torch.exp2(s[:128].max() - m2)
    l = torch.exp2(s[:128] - s[:128].max()).sum() * a + torch.exp2(s[128:] - m2).sum()
    want = (a * (p1 @ v[0, :128, 0].to(F64)) + p2 @ v[0, 128:, 0].to(F64)) / l
    assert torch.allclose(pre[0, 0, 0], want, rtol=1e-14, atol=1e-15)
    assert abs(float(lse[0, 0, 0]) - float((m2 + torch.log2(l)) * R.LN2)) < 1e-14


# ------------------------------------------------------------------------------------------------ the probes
@pytest.mark.parametrize("case", SMALL, ids=[c.id for c in SMALL])
def test_probe_closed_forms_equal_the_restatement(case):
    inp = R.make_inputs(case, probe="fwd")
    pre, lse, _ = R.fwd_case(case, inp)
    e_out, e_lse = R.probe_fwd_case(case, inp)
    assert torch.equal(R.bf16r(pre), e_out)
    assert torch.equal(torch.isinf(lse), torch.isinf(e_lse))
    fin = torch.isfinite(e_lse)
    assert torch.allclose(lse[fin], e_lse[fin], rtol=1e-14, atol=1e-14)
    assert bool(fin.any())
    if not case.has_bwd:
        return
    for probe in ("bwd_q", "bwd_k"):
        inp = R.make_inputs(case, probe=probe)
        lead = (1, case.S) if case.kind == "packed" else (case.B, case.S)
        (dq, dk, dv), _ = R.bwd_case(case, inp, torch.zeros(*lead, case.nh * case.d), torch.zeros(lead[0], case.nh, case.S))
        e = R.probe_bwd_case(case, inp)
        for got, want in zip((dq, dk, dv), e):
            assert torch.equal(R.bf16r(got), want)
        nz = e[0] if probe == "bwd_q" else e[1]
        assert bool((nz != 0).any())


# ------------------------------------------------------------------------------------------------ injected faults
FWD = "fwd"
BWD = "bwd"
# fault -> (the kernels it lives in, candidate cases)
FAULTS = {
    "diag_wg1": (FWD, [_find(kind="self", S=129, d=64, causal=True, nh=2, nkv=2, dist="normal")]),
    "coff": (FWD, [_find(kind="cache", S=5, mask=True)]),
    "tile_first": (FWD, [_find(kind="self", S=257, d=64, causal=False, nh=2, nkv=2, dist="normal", scale=None)]),
    "tile_last": (FWD, [_find(kind="self", S=257, d=64, causal=False, nh=2, nkv=2, dist="normal", scale=None)]),
    "kv_tail": (FWD, [_find(kind="cross", S=64, Skv=77)]),
    "mask_b1": (FWD, [_find(kind="cache", S=5, mask=True)]),
    "gqa_mod": (FWD + BWD, [_find(kind="self", nh=8, nkv=4)]),
    "alpha_l": (FWD, [_find(kind="self", S=384, causal=True, dist="rise")]),
    "lse_log2": (FWD, [_find(kind="self", S=65, d=128, causal=True, nh=2, nkv=2)]),
    "dkdv_i0": (BWD, [_find(kind="self", S=129, d=64, causal=True, nh=2, nkv=2, dist="normal")]),
    "dq_kvend": (BWD, [_find(kind="self", S=129, d=64, causal=True, nh=2, nkv=2, dist="normal")]),
    "dkv_group": (BWD, [_find(kind="self", nh=8, nkv=4)]),
    "packed_tail": (FWD, [_find(kind="packed", d=128, causal=False)]),
}


def _rejects(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


def _rejected_by(case, fault, where):
    """Names of the checks (at 10x their constants) that reject `fault` injected into the restatement on the case's own inputs."""
    hits = []
    inp = R.make_inputs(case)
    pre, lse, mass = R.fwd_case(case, inp)
    if FWD in where:
        fpre, flse, _ = R.fwd_case(case, inp, fault=fault)
        if _rejects(lambda: R.check_out(R.bf16r(fpre), pre, mass, c=10 * R.C_ACC)):
            hits.append("out bound")
        if _rejects(lambda: R.check_lse(flse.to(F32), lse, c=10 * R.C_LSE)):
            hits.append("lse bound")
        pin = R.make_inputs(case, probe="fwd")
        e_out, e_lse = R.probe_fwd_case(case, pin)
        fo, fl, _ = R.fwd_case(case, pin, fault=fault)
        fin = torch.isfinite(e_lse)
        if (not torch.equal(torch.isinf(fl), ~fin)
                or bool((((fl - e_lse).abs() / (1 + e_lse.abs()))[fin] > 10 * R.PROBE_LSE_TOL).any())
                or bool(((R.bf16r(fo) - e_out).abs() > 10 * R.ulp(e_out)).any())):
            hits.append("forward probe")
    if BWD in where and case.has_bwd:
        o, l32 = R.bf16r(pre).to(torch.bfloat16), lse.to(F32)
        good, masses = R.bwd_case(case, inp, o, l32)
        bad, _ = R.bwd_case(case, inp, o, l32, fault=fault)
        for n, g, b, m in zip(("dq", "dk", "dv"), good, bad, masses):
            if _rejects(lambda: R.check_out(R.bf16r(b), g, m, c=10 * R.C_ACC)):
                hits.append(f"{n} bound")
        lead = (1, case.S) if case.kind == "packed" else (case.B, case.S)
        for probe in ("bwd_q", "bwd_k"):
            pin = R.make_inputs(case, probe=probe)
            zo, zl = torch.zeros(*lead, case.nh * case.d), torch.zeros(lead[0], case.nh, case.S)
            e = R.probe_bwd_case(case, pin)
            fb, _ = R.bwd_case(case, pin, zo, zl, fault=fault)
            if any(not torch.equal(R.bf16r(x), y) for x, y in zip(fb, e)):
                hits.append(f"{probe} probe")
    return hits


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_comparison_rejects_injected_fault(fault):
    where, cases = FAULTS[fault]
    found = {c.id: _rejected_by(c, fault, where) for c in cases}
    print(f"fault {fault}: {found}")
    assert any(found.values()), f"{fault} passes every check at 10x slack: {found}"


# ------------------------------------------------------------------------------------------------ an fp32 emulation passes
@pytest.mark.parametrize("case", SMALL, ids=[c.id for c in SMALL])
def test_fp32_emulation_passes(case):
    inp = R.make_inputs(case)
    pre, lse, mass = R.fwd_case(case, inp)
    epre, else_, _ = R.fwd_case(case, inp, dt=F32)
    R.check_out(R.bf16r(epre.to(F64)), pre, mass, what=f"{case.id} emulated out")
    R.check_lse(else_, lse, what=f"{case.id} emulated lse")
    if not case.has_bwd:
        return
    o = R.bf16r(epre.to(F64)).to(torch.bfloat16)
    good, masses = R.bwd_case(case, inp, o, else_)
    emu, _ = R.bwd_case(case, inp, o, else_, dt=F32)
    for n, g, e, m in zip(("dq", "dk", "dv"), good, emu, masses):
        R.check_out(R.bf16r(e.to(F64)), g, m, what=f"{case.id} emulated {n}")

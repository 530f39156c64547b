"""The flash-attention kernels of csrc/attn_sm90.cu (forward, backward prep, dK/dV, dQ) against their float64 restatements
(oracle/attn_oracle.py), element by element, through every public entry: `attn_fwd` (fused qkv, right padding, GQA), `attn_fwd_cross_lse`,
`attn_fwd_cache` (bottom-right causal mask, kv_rows > Skv, kv_mask), `attn_fwd_varlen`, `attn_bwd`, `attn_bwd_cross` and
`attn_bwd_varlen`, at every geometry of attn_oracle.CASES.

Criterion (`check_out`): every bf16 element within one ulp + C_ACC x term mass of the rounded restatement, except at most 0.1 % (bf16
ties of P or dS that fp32 rounded the other way) within one ulp + 2^-8 x term mass; at most 1 % differ at all; elements with no term
are exactly 0.  lse within C_LSE (1 + |lse|), +inf exactly on rows with no visible key.  The probes compare counts and integer sums
bit for bit (the forward's out to one ulp, its 1 / l being approximate), and every output is written into a view of a wider buffer
whose other elements must keep a sentinel.
"""
import pytest
import torch

from oracle import attn_oracle as R

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64
SENT = 12352.0        # bf16-exact sentinel
PAD = 64              # sentinel columns right of every output view


def _ops():
    from dreamllm_b200 import ops
    return ops


def _L():
    from dreamllm_b200._lib import lib
    return lib()


def _p(t):
    return 0 if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(inp):
    return {k: v.cuda() for k, v in inp.items()}


def _views(case, inp):
    """(q, k, v) device views in the entry's layout (re-sliced from the device copies of the underlying buffers)."""
    nh, nkv, d = case.nh, case.nkv, case.d
    if case.kind in ("self", "packed"):
        return tuple(R.split_heads(inp["qkv"], (nh, nkv, nkv), d))
    if case.kind == "cross":
        return (inp["q"], *R.split_heads(inp["kv"], (nkv, nkv), d))
    return inp["q"], inp["kc"], inp["vc"]


def _fwd(case, inp):
    """(out, lse) through the case's public forward entry."""
    ops = _ops()
    q, k, v = _views(case, inp)
    sc = case.scale
    if case.kind == "self":
        return ops.attn_fwd(q, k, v, causal=case.causal, seqlens=inp.get("seqlens"), scale=sc)
    if case.kind == "cross":
        return ops.attn_fwd_cross_lse(q, k, v, scale=sc)
    if case.kind == "cache":
        return ops.attn_fwd_cache(q, k, v, case.Skv, causal=True, scale=sc, kv_mask=inp.get("mask"), return_lse=True)
    return ops.attn_fwd_varlen(q, k, v, inp["cu"], case.max_seqlen, causal=case.causal, scale=sc)


def _fwd_wide(case, inp):
    """The forward through the C entry with out a view of a wider buffer prefilled with the sentinel: (buffer, view, lse)."""
    q, k, v = _views(case, inp)
    nh, nkv, d = case.nh, case.nkv, case.d
    lead = (case.S,) if case.kind == "packed" else (case.B, case.S)
    buf = torch.full((*lead, nh * d + PAD), SENT, dtype=BF, device="cuda")
    view = buf[..., :nh * d]
    ld_o = nh * d + PAD
    if case.kind == "packed":
        lse = torch.empty(nh, case.S, dtype=torch.float32, device="cuda")
        rc = _L().dllm_attn_fwd_varlen(_p(q), _p(k), _p(v), _p(view), _p(lse), _p(inp["cu"]), case.B, case.S, case.max_seqlen, nh, nkv,
                                       d, q.stride(0), k.stride(0), ld_o, int(case.causal), case.scale_v, _stream())
    else:
        lse = torch.empty(case.B, nh, case.S, dtype=torch.float32, device="cuda")
        mask = inp.get("mask")
        rc = _L().dllm_attn_fwd_gqa(_p(q), _p(k), _p(v), _p(view), _p(lse), _p(inp.get("seqlens")), _p(mask),
                                    0 if mask is None else mask.stride(0), case.B, case.S, case.keys, k.shape[1], nh, nkv, d,
                                    q.stride(1), k.stride(1), ld_o, int(case.causal), case.scale_v, _stream())
    assert rc == 0, rc
    return buf, view, lse


def _bwd(case, inp, out, lse, dout):
    """(bufs, dq, dk, dv) through the case's public backward entry, the gradients written into views of sentinel-filled buffers."""
    ops = _ops()
    q, k, v = _views(case, inp)
    nh, nkv, d = case.nh, case.nkv, case.d
    sc = case.scale
    if case.kind == "cross":
        bq = torch.full((case.B, case.S, nh * d + PAD), SENT, dtype=BF, device="cuda")
        bkv = torch.full((case.B, case.Skv, 2 * nkv * d + PAD), SENT, dtype=BF, device="cuda")
        (dq,), (dk, dv) = R.split_heads(bq, (nh,), d), R.split_heads(bkv, (nkv, nkv), d)
        ops.attn_bwd_cross(dout, q, k, v, out, lse, dq, dk, dv, scale=sc)
        return (bq, bkv), dq, dk, dv
    lead = (case.S,) if case.kind == "packed" else (case.B, case.S)
    W = (nh + 2 * nkv) * d
    buf = torch.full((*lead, W + PAD), SENT, dtype=BF, device="cuda")
    dq, dk, dv = R.split_heads(buf, (nh, nkv, nkv), d)
    if case.kind == "self":
        ops.attn_bwd(dout, q, k, v, out, lse, dq, dk, dv, causal=case.causal, seqlens=inp.get("seqlens"), scale=sc)
    else:
        ops.attn_bwd_varlen(dout, q, k, v, out, lse, dq, dk, dv, inp["cu"], case.max_seqlen, causal=case.causal, scale=sc)
    return (buf,), dq, dk, dv


def _sentinel_kept(bufs, views, what):
    for buf in bufs:
        keep = torch.ones_like(buf, dtype=torch.bool)
        for v in views:
            if v.untyped_storage().data_ptr() == buf.untyped_storage().data_ptr():
                keep.view(-1)[torch.as_strided(torch.arange(buf.numel(), device="cuda"), v.shape, v.stride(),
                                                v.storage_offset() - buf.storage_offset()).flatten()] = False
        assert bool((buf[keep] == SENT).all()), f"{what}: {int((buf[keep] != SENT).sum())} elements outside the views were written"


def _shape_out(case, t):
    return t.reshape(1 if case.kind == "packed" else case.B, case.S, case.nh, case.d)


def _shape_lse(case, t):
    return t.reshape(1 if case.kind == "packed" else case.B, case.nh, case.S)


def _shape_kv(case, t):
    return t.reshape(1 if case.kind == "packed" else case.B, case.keys, case.nkv, case.d)


def _report(case, name, frac):
    """The slack this output needed, as a fraction of its constant (C_ACC, or C_LSE for lse): printed for calibration."""
    print(f"attn slack {case.id} {name}: {frac:.4f}")


# ------------------------------------------------------------------------------------------------ float64 parity
@pytest.mark.parametrize("case", R.CASES, ids=[c.id for c in R.CASES])
def test_attn_vs_float64(case):
    host = R.make_inputs(case)
    inp = _dev(host)
    out, lse = _fwd(case, inp)
    buf, view, lse_w = _fwd_wide(case, inp)
    torch.cuda.synchronize()
    assert torch.equal(view, out) and torch.equal(lse_w, lse), "a wider output stride changed the result"
    _sentinel_kept([buf], [view], f"{case.id} out")

    pre, lse_ref, mass = R.fwd_case(case, host, device="cuda")
    _report(case, "out", R.slack_needed(_shape_out(case, out), pre, mass) / R.C_ACC)
    _report(case, "lse", R.lse_slack_needed(_shape_lse(case, lse), lse_ref) / R.C_LSE)
    R.check_out(_shape_out(case, out), pre, mass, what=f"{case.id} out")
    R.check_lse(_shape_lse(case, lse), lse_ref, what=f"{case.id} lse")

    if case.kind == "cache":                               # the rows past Skv are never read: zeros there give the same bits
        z = dict(inp)
        for n in ("kc", "vc"):
            z[n] = inp[n].clone()
            z[n][:, case.Skv:] = 0
        out0, lse0 = _fwd(case, z)
        assert torch.equal(out0, out) and torch.equal(lse0, lse), "kv-cache rows past Skv changed the result"
    if case.has_bwd:
        dout = inp["dout"]
        bufs, dq, dk, dv = _bwd(case, inp, out, lse, dout)
        torch.cuda.synchronize()
        _sentinel_kept(bufs, [dq, dk, dv], f"{case.id} dqkv")
        (rq, rk, rv), (mq, mk, mv) = R.bwd_case(case, host, out, lse, device="cuda")
        for name, got, ref, m, shp in (("dq", dq, rq, mq, _shape_out), ("dk", dk, rk, mk, _shape_kv), ("dv", dv, rv, mv, _shape_kv)):
            _report(case, name, R.slack_needed(shp(case, got), ref, m) / R.C_ACC)
            R.check_out(shp(case, got), ref, m, what=f"{case.id} {name}")


# ------------------------------------------------------------------------------------------------ exact probes
def test_exp2_of_zero_is_one():
    """The probes rely on ex2.approx(0) == 1: one visible key with q = 0 gives a weight of exactly 1, so out = v and lse = 0."""
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    for d in (64, 128):
        qkv = torch.zeros(1, 1, 3 * d, dtype=BF)
        qkv[..., d:] = torch.randn(1, 1, 2 * d, generator=g).to(BF)
        qkv = qkv.cuda()
        q, k, v = R.split_heads(qkv, (1, 1, 1), d)
        out, lse = ops.attn_fwd(q, k, v, causal=True)
        assert torch.equal(out.view(-1), v.reshape(-1)), d
        assert float(lse) == 0.0, float(lse)


@pytest.mark.parametrize("case", R.CASES, ids=[c.id for c in R.CASES])
def test_attn_probes(case):
    # forward: q = 0, every visible weight exactly 1 -> lse = ln(count), out = sum of the visible v / count
    host = R.make_inputs(case, probe="fwd")
    inp = _dev(host)
    out, lse = _fwd(case, inp)
    e_out, e_lse = R.probe_fwd_case(case, host, device="cuda")
    got, gl = _shape_out(case, out).to(F64), _shape_lse(case, lse).to(F64)
    fin = torch.isfinite(e_lse)
    assert bool((gl[~fin] == R.INF).all()), f"{case.id}: lse not +inf on a row with no visible key"
    assert bool((got.permute(0, 2, 1, 3)[~fin] == 0).all()), f"{case.id}: out not 0 on a row with no visible key"
    lerr = ((gl - e_lse).abs() / (1 + e_lse.abs()))[fin]
    assert bool((lerr <= R.PROBE_LSE_TOL).all()), f"{case.id}: probe lse off by {float(lerr.max()):.3g} (1 + |lse|)"
    oerr = (got - e_out).abs() / R.ulp(e_out)
    assert bool((oerr <= 1).all()), f"{case.id}: probe out off by {float(oerr.max())} ulp on {int((oerr > 1).sum())} elements"
    if not case.has_bwd:
        return
    # backward: lse = 0, O = 0 -> P = 1 on every kept pair, delta = 0; q = 0 pins dV and dQ, k = 0 pins dV and dK, bit for bit
    for probe, names in (("bwd_q", ("dq", "dv")), ("bwd_k", ("dk", "dv"))):
        host = R.make_inputs(case, probe=probe)
        inp = _dev(host)
        zo = torch.zeros_like(inp["dout"])
        zl = torch.zeros_like(lse)
        bufs, dq, dk, dv = _bwd(case, inp, zo, zl, inp["dout"])
        torch.cuda.synchronize()
        _sentinel_kept(bufs, [dq, dk, dv], f"{case.id} {probe}")
        exp = dict(zip(("dq", "dk", "dv"), R.probe_bwd_case(case, host, device="cuda")))
        got = {"dq": _shape_out(case, dq), "dk": _shape_kv(case, dk), "dv": _shape_kv(case, dv)}
        for n in names:
            diff = got[n].to(F64) != exp[n]
            assert not bool(diff.any()), f"{case.id} {probe} {n}: {int(diff.sum())} of {diff.numel()} elements differ"

"""TEST INFRASTRUCTURE ONLY — float64 restatements of the flash-attention kernels of csrc/attn_sm90.cu (forward, backward prep, dK/dV,
dQ), reached through `ops.attn_fwd`, `attn_fwd_cross_lse`, `attn_fwd_cache`, `attn_fwd_varlen`, `attn_bwd`, `attn_bwd_cross` and
`attn_bwd_varlen`.

Plain torch (no `dreamllm_b200` import); every function runs on whatever device its inputs live on.  The kernels compute in fp32 from
bf16 operands and round to bf16 at fixed points; the restatements do the same walk in float64 and round at the same points:
  * forward (attn_fwd_kernel): keys in 128-key tiles; running max m in log2 units with the kernel's fp32 scale_log2 = fl32(scale log2 e);
    alpha = 0 while m is -inf, exp2(m_old - m_new) after; P rounded to bf16 relative to the running max of its tile (acc_to_afrag);
    l sums the unrounded p; out = bf16(sum bf16(P) V / l); lse = (m + log2 l) ln 2, +inf on rows with no visible key and rows >= q_len,
    whose out is 0;
  * backward (prep + dK/dV + dQ), given the kernel's own O and lse: P = exp2(s scale_log2 - fl32(lse log2 e)) on the pairs each kernel
    keeps; delta = sum dO O; dV = bf16(sum bf16(P) dO); dS = bf16(P (dP - delta)); dQ = bf16(fl32(scale) sum dS K) and
    dK = bf16(fl32(scale) sum dS Q); under GQA dK / dV sum the group's q heads.
Each output comes with its term mass (the sum of the absolute values of the terms, normalised as the output is), which scales the
fp32 accumulation slack of the comparison.  The probes pin the visibility rules bit for bit: with q = 0 every visible weight is exactly
1 (ex2.approx(0) == 1), so the forward is a count and a sum; with lse = 0 and O = 0 the backward is integer arithmetic.

The geometry table, the seeded inputs and the comparison used by tests/test_attn_float64_gpu.py live here too, so that
tests/test_attn_float64_cpu.py can show on the very same inputs that the comparison rejects a kernel that is subtly wrong.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from oracle.conv3x3_oracle import bf16r, ulp

BF = torch.bfloat16
F64 = torch.float64
F32 = torch.float32
LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453
INF = float("inf")

# Per-element fp32 slack of the kernels, as a fraction of the term mass (forward: sum bf16(P) |V| / l; dV: sum bf16(P) |dO|; dQ / dK:
# scale sum P (|dO| |V| + |dO| |O|) |K| resp. |Q|, which also bounds the fp32 error of dP - delta).  The largest needed on an H100 80GB
# HBM3 (700 W) over every case of CASES was 8.1e-7 (dV, self-full-d64-B2-h2g1-S577-kt5-rise); the others: dQ 4.4e-8, dK 2.3e-8, and
# out 0 (every forward output within one ulp, bar the allowed flips).  2^-18 = 3.8e-6 leaves 4.7x.
C_ACC = 2.0 ** -18
# lse (fp32) within C_LSE (1 + |lse|) of the float64 value.  The largest needed on the same card was 4.5e-7 (the sharp-softmax
# self-causal-d128-B2-h2g1-S384-kt3-sharp); 2^-19 = 1.9e-6 leaves 4.3x.
C_LSE = 2.0 ** -19
# forward probe: lse = ln(count) within this many times (1 + |lse|) (lg2.approx and one fp32 multiply)
PROBE_LSE_TOL = 2.0 ** -20
FLIP_FRAC = 1e-3          # at most this fraction of elements beyond ulp + C_ACC mass (bf16 ties of P or dS rounded the other way) ...
FLIP_SLACK = 2.0 ** -8    # ... and those within ulp + FLIP_SLACK mass (one rounding step of the weights)
DIFF_FRAC = 1e-2          # at most this fraction of elements differ from the rounded reference at all


def fl32(x: float) -> float:
    return float(torch.tensor(x, dtype=F32))


def _rb(x, rnd=True):
    """bf16 rounding point (identity with rounding switched off); keeps x's dtype."""
    return x.to(F32).to(BF).to(x.dtype) if rnd else x


def kv_head_map(nh: int, nkv: int, fault: str | None = None) -> torch.Tensor:
    """kv head each q head reads: h / group (reference repeat_kv).  Fault "gqa_mod": h % nkv."""
    h = torch.arange(nh)
    return h % nkv if fault == "gqa_mod" else h // (nh // nkv)


# ------------------------------------------------------------------------------------------------ visibility
def visibility(B, S, Skv, causal, seqlens=None, kv_mask=None, fault=None):
    """(vis [B, S, Skv] bool, qrow [B, S] bool) of attn_fwd_kernel: key j is visible to row i iff j < kv_len, kv_mask[b, j] != 0 and
    (causal) j <= i + coff, coff = Skv - S (bottom-right aligned), for rows i < q_len.  kv_len = min(seqlens[b], Skv) and q_len = kv_len
    with right padding (seqlens), else Skv and S.  Faults: "diag_wg1" (the diagonal one key late on the second warpgroup's rows,
    i % 128 >= 64), "coff" (coff one short), "tile_first" / "tile_last" (key 128 t, resp. 128 t + 127, dropped), "mask_b1" (batch
    entry 1's kv_mask ignored)."""
    if seqlens is not None:
        kv_len = torch.tensor([min(int(s), Skv) for s in seqlens])
        q_len = kv_len
    else:
        kv_len, q_len = torch.full((B,), Skv), torch.full((B,), S)
    i = torch.arange(S)[:, None]
    j = torch.arange(Skv)[None, :]
    vis = (j[None] < kv_len[:, None, None]).expand(B, S, Skv).clone()
    if kv_mask is not None:
        m = kv_mask[:, :Skv].bool().clone()
        if fault == "mask_b1" and B > 1:
            m[1] = True
        vis &= m[:, None, :]
    if causal:
        coff = Skv - S - (1 if fault == "coff" else 0)
        lim = i + coff + ((i % 128 >= 64).long() if fault == "diag_wg1" else 0)
        vis &= (j <= lim)[None]
    if fault == "tile_first":
        vis &= (j % 128 != 0)[None]
    if fault == "tile_last":
        vis &= (j % 128 != 127)[None]
    qrow = torch.arange(S)[None, :] < q_len[:, None]
    return vis & qrow[:, :, None], qrow


def bwd_masks(vis, causal, fault=None):
    """(vis_dq, vis_kv): the pairs the dQ and dK/dV kernels keep (both = vis).  Faults: "dkdv_i0" (the dK/dV CTA of kv tile kv0 starts
    at q tile kv0 / 64 + 1: q rows [kv0, kv0 + 64) drop out of its keys' sums), "dq_kvend" (dQ's kv_end one key short: key
    128 (i / 128) + 127 drops out of row i's sum)."""
    S, Skv = vis.shape[1:]
    i = torch.arange(S, device=vis.device)[:, None]
    j = torch.arange(Skv, device=vis.device)[None, :]
    vis_dq, vis_kv = vis, vis
    if causal and fault == "dkdv_i0":
        vis_kv = vis & ~(i // 64 == 2 * (j // 128))[None]
    if causal and fault == "dq_kvend":
        vis_dq = vis & ~(j == (i // 128) * 128 + 127)[None]
    return vis_dq, vis_kv


# ------------------------------------------------------------------------------------------------ restatements
def _heads(x, hm, dt):
    """[B, L, nkv, d] -> [B, nh, L, d] through the head map."""
    return x.to(dt)[:, :, hm.to(x.device)].permute(0, 2, 1, 3)


def fwd_ref(q, k, v, vis, qrow, scale, kv_head=None, dt=F64, rnd=True, fault=None, tile=128):
    """attn_fwd_kernel on one dense problem: q [B, S, nh, d], k / v [B, Skv, nkv, d], vis / qrow from `visibility`.  Returns
    (pre [B, S, nh, d], lse [B, nh, S], mass [B, S, nh, d]): out = bf16(pre).  dt = float32 with rnd=True emulates the kernel's
    arithmetic; rnd=False drops every rounding point (plain softmax attention).  Faults: "alpha_l" (alpha rescales o but not l),
    "lse_log2" (lse left in log2 units)."""
    B, S, nh, d = q.shape
    hm = kv_head if kv_head is not None else kv_head_map(nh, k.shape[2])
    qd = q.to(dt).permute(0, 2, 1, 3)
    kd, vd = _heads(k, hm, dt), _heads(v, hm, dt)
    c = fl32(scale * LOG2E) if rnd else scale * LOG2E
    s = (qd @ kd.transpose(-1, -2)).masked_fill(~vis[:, None].to(q.device), -INF) * c
    m = torch.full((B, nh, S), -INF, dtype=dt, device=q.device)
    l = torch.zeros_like(m)
    o = torch.zeros(B, nh, S, d, dtype=dt, device=q.device)
    oa = torch.zeros_like(o)
    zero = torch.zeros((), dtype=dt, device=q.device)
    for j0 in range(0, k.shape[1], tile):
        sj = s[..., j0:j0 + tile]
        m_new = torch.maximum(m, sj.amax(-1))
        alpha = torch.where(m == -INF, zero, torch.exp2(m - m_new))
        m_use = torch.where(m_new == -INF, zero, m_new)
        p = torch.exp2(sj - m_use[..., None])
        l = (l if fault == "alpha_l" else l * alpha) + p.sum(-1)
        pb = _rb(p, rnd)
        vj = vd[:, :, j0:j0 + tile]
        o = o * alpha[..., None] + pb @ vj
        oa = oa * alpha[..., None] + pb @ vj.abs()
        m = m_new
    ok = qrow[:, None, :].to(q.device) & (l > 0)
    inv = torch.where(ok, 1.0 / l.clamp_min(1e-300), zero)
    lse = (m + torch.log2(l.clamp_min(1e-300))) * (1.0 if fault == "lse_log2" else LN2)
    lse = torch.where(ok, lse, torch.full_like(lse, INF))
    return (o * inv[..., None]).permute(0, 2, 1, 3), lse, (oa * inv[..., None]).permute(0, 2, 1, 3)


def bwd_ref(q, k, v, o, lse, do, vis_dq, vis_kv, qrow, scale, kv_head=None, dkv_heads=None, dt=F64, rnd=True):
    """attn_bwd_prep + dK/dV + dQ on one dense problem, from the kernel's own o [B, S, nh, d] and lse [B, nh, S].  Returns
    ((dq, dk, dv) before rounding, (mass_dq, mass_dk, mass_dv)), dq [B, S, nh, d] and dk / dv [B, Skv, nkv, d].  dkv_heads (bool [nh],
    default all) selects the q heads whose terms dK / dV sum (fault: only group - 1 of them)."""
    B, S, nh, d = q.shape
    Skv, nkv = k.shape[1], k.shape[2]
    dev = q.device
    hm = (kv_head if kv_head is not None else kv_head_map(nh, nkv)).to(dev)
    qd, dod, od = (x.to(dt).permute(0, 2, 1, 3) for x in (q, do, o))
    kd, vd = _heads(k, hm, dt), _heads(v, hm, dt)
    c = fl32(scale * LOG2E) if rnd else scale * LOG2E
    sc = fl32(scale) if rnd else scale
    l2 = (lse.to(dev).to(F32) * torch.tensor(LOG2E, dtype=F32, device=dev)).to(dt) if rnd else lse.to(dev).to(dt) * LOG2E
    x = (qd @ kd.transpose(-1, -2)) * c - l2[..., None]
    rows = qrow[:, None, :, None].to(dev)
    zero = torch.zeros((), dtype=dt, device=dev)
    e = torch.exp2(torch.where(rows, x, zero))
    delta = (dod * od).sum(-1, keepdim=True)
    mdelta = (dod * od).abs().sum(-1, keepdim=True)
    dp = dod @ vd.transpose(-1, -2)
    mp = dod.abs() @ vd.abs().transpose(-1, -2) + mdelta
    out, mass = [], []
    for vis in (vis_dq, vis_kv):
        p = torch.where(vis[:, None].to(dev) & rows, e, zero)
        out.append((p, _rb(p * (dp - delta), rnd), p * mp))
    (_, ds_q, ms_q), (p_k, ds_k, ms_k) = out
    dq = sc * (ds_q @ kd)
    mdq = sc * (ms_q @ kd.abs())
    w = torch.ones(nh, dtype=dt, device=dev) if dkv_heads is None else dkv_heads.to(dev).to(dt)
    w = w[None, :, None, None]
    pb = _rb(p_k, rnd)
    per_h = [sc * (ds_k.transpose(-1, -2) @ qd), sc * (ms_k.transpose(-1, -2) @ qd.abs()),
             pb.transpose(-1, -2) @ dod, pb.transpose(-1, -2) @ dod.abs()]
    red = []
    for t in per_h:                                    # [B, nh, Skv, d] -> [B, Skv, nkv, d], summed over each kv head's q heads
        acc = torch.zeros(B, nkv, Skv, d, dtype=dt, device=dev)
        acc.index_add_(1, hm, t * w)
        red.append(acc.permute(0, 2, 1, 3))
    dk, mdk, dv, mdv = red
    return (dq.permute(0, 2, 1, 3), dk, dv), (mdq.permute(0, 2, 1, 3), mdk, mdv)


# ------------------------------------------------------------------------------------------------ the comparison
def slack_needed(got, pre, mass):
    """Smallest c with |got - bf16(pre)| <= ulp + c mass at all but the allowed flips (FLIP_FRAC of the elements)."""
    got = got.to(pre.device).to(F64)
    y = bf16r(pre)
    excess = ((got - y).abs() - ulp(y)) / mass.clamp_min(1e-300)
    excess = excess.clamp_min(0.0).flatten()
    k = int(FLIP_FRAC * excess.numel())
    return float(excess.kthvalue(excess.numel() - k).values) if excess.numel() > k else 0.0


def check_out(got, pre, mass, c=C_ACC, what=""):
    """Raise AssertionError unless the kernel's bf16 `got` matches y = bf16(pre): every element within ulp(y) + c mass, except at most
    FLIP_FRAC of them (a bf16 tie of P or dS that fp32 rounded the other way) which are within ulp(y) + FLIP_SLACK mass; and at most
    DIFF_FRAC of the elements differ from y at all, not counting those whose unrounded value lies within c mass of a rounding midpoint
    (dQ / dK of a row whose dP - delta cancels, such as a row with a single visible key, is rounding noise around 0)."""
    got = got.to(pre.device).to(F64).reshape(pre.shape)
    y = bf16r(pre)
    err = (got - y).abs()
    u = ulp(y)
    empty = mass == 0                                  # no term at all (masked rows, padding): exactly 0
    assert bool((got[empty] == 0).all()), f"{what}: {int((got[empty] != 0).sum())} elements with no visible term are not 0"
    flip = ~(err <= u + c * mass)                      # NaN counts as a flip
    n = err.numel()
    nf = int(flip.sum())
    if nf:
        far = flip & ~(err <= u + FLIP_SLACK * mass)
        if bool(far.any()) or nf > FLIP_FRAC * n:
            bad = far if bool(far.any()) else flip
            i = int(bad.flatten().nonzero()[0])
            idx = tuple(int(t) for t in torch.unravel_index(torch.tensor(i), y.shape))
            raise AssertionError(f"{what}: {nf} of {n} elements beyond ulp + c mass (c = {c:.3g}), {int(far.sum())} beyond ulp + "
                                 f"2^-8 mass; first at {idx}: got {float(got.flatten()[i])}, reference {float(y.flatten()[i])}, "
                                 f"mass {float(mass.flatten()[i]):.3g}")
    near = u / 2 - (pre - y).abs() <= c * mass       # the fp32 slack reaches a rounding midpoint: either neighbour is right
    frac = float(((err > 0) & ~near).double().mean())
    assert frac <= DIFF_FRAC, f"{what}: {frac:.4f} of the elements differ from the reference (at most {DIFF_FRAC})"


def lse_slack_needed(got, ref):
    got = got.to(ref.device).to(F64)
    fin = torch.isfinite(ref)
    if not bool(fin.any()):
        return 0.0
    return float(((got - ref).abs() / (1 + ref.abs()))[fin].max())


def check_lse(got, ref, c=C_LSE, what=""):
    """lse (fp32): +inf exactly where the reference is +inf, elsewhere within c (1 + |ref|)."""
    got = got.to(ref.device).to(F64).reshape(ref.shape)
    fin = torch.isfinite(ref)
    assert bool((got[~fin] == INF).all()), f"{what}: lse not +inf on {int((got[~fin] != INF).sum())} rows with no visible key"
    err = ((got - ref).abs() / (1 + ref.abs()))[fin]
    ok = err <= c
    if not bool(ok.all()):
        raise AssertionError(f"{what}: lse off by up to {float(err.nan_to_num(INF).max()):.3g} (1 + |lse|), bound {c:.3g}, on "
                             f"{int((~ok).sum())} of {ok.numel()} rows")


# ------------------------------------------------------------------------------------------------ probes (closed forms)
def probe_fwd_expect(v, vis, qrow, kv_head):
    """q = 0: every visible weight is exactly 1.  (out [B, S, nh, d] as float64 of bf16(sum_visible v / count), 0 on rows without a
    visible key; lse [B, nh, S] = ln(count), +inf there)."""
    hm = kv_head.to(v.device)
    cnt = vis.to(v.device).to(F64).sum(-1)                             # [B, S]
    sv = vis.to(v.device).to(F64)[:, None] @ _heads(v, hm, F64)       # [B, nh, S, d]
    ok = (cnt > 0) & qrow.to(v.device)
    out = torch.where(ok[:, None, :, None], bf16r(sv / cnt.clamp_min(1)[:, None, :, None]), torch.zeros((), dtype=F64, device=v.device))
    lse = torch.where(ok, torch.log(cnt.clamp_min(1)), torch.full_like(cnt, INF))
    return out.permute(0, 2, 1, 3), lse[:, None].expand(-1, hm.numel(), -1)


def probe_bwd_expect(q, k, v, do, vis_dq, vis_kv, qrow, scale, kv_head):
    """lse = 0, O = 0 and q k^T = 0 (q = 0 or k = 0): P = 1 on the kept pairs, delta = 0, dS = dP = dO V^T, all integers below 2^24.
    Returns bf16 (dq, dk, dv) as float64, each bf16(fl32(integer sum) * fl32(scale)) (dv unscaled)."""
    B, S, nh, d = q.shape
    nkv = k.shape[2]
    dev = q.device
    hm = kv_head.to(dev)
    qd, dod = (x.to(F64).permute(0, 2, 1, 3) for x in (q, do))
    kd, vd = _heads(k, hm, F64), _heads(v, hm, F64)
    dp = dod @ vd.transpose(-1, -2)
    rows = qrow[:, None, :, None].to(dev)
    mq = (vis_dq[:, None].to(dev) & rows).to(F64)
    mk = (vis_kv[:, None].to(dev) & rows).to(F64)
    sc = torch.tensor(scale, dtype=F32, device=dev)

    def fin(acc, mul):
        return ((acc.to(F32) * mul) if mul is not None else acc.to(F32)).to(BF).to(F64)
    dq = fin((mq * dp) @ kd, sc).permute(0, 2, 1, 3)
    red = []
    for t in ((mk * dp).transpose(-1, -2) @ qd, mk.transpose(-1, -2) @ dod):
        acc = torch.zeros(B, nkv, k.shape[1], d, dtype=F64, device=dev)
        acc.index_add_(1, hm, t)
        red.append(acc.permute(0, 2, 1, 3))
    return dq, fin(red[0], sc), fin(red[1], None)


# ------------------------------------------------------------------------------------------------ geometries
@dataclass(frozen=True)
class Case:
    kind: str                       # self (fused qkv, optional right padding) | cross | cache | packed
    B: int
    S: int                          # query rows (packed: T)
    nh: int
    nkv: int
    d: int
    causal: bool = False
    Skv: int = 0                    # cross / cache: keys (cache: past + S)
    seqlens: tuple | None = None    # self: right padding
    mask: bool = False              # cache: kv_mask, odd batch entries left-padded
    lens: tuple | None = None       # packed: sample lengths
    max_seqlen: int = 0             # packed
    scale: float | None = None
    dist: str = "normal"            # normal | sharp (logit sd ~10) | rise / fall (row max rises / falls on every key tile)
    tag: str = ""

    @property
    def keys(self) -> int:
        return self.S if self.kind in ("self", "packed") else self.Skv

    @property
    def scale_v(self) -> float:
        return self.d ** -0.5 if self.scale is None else self.scale

    @property
    def has_bwd(self) -> bool:
        return self.kind != "cache"

    @property
    def id(self) -> str:
        c = "causal" if self.causal else "full"
        kt = -(-self.keys // 128)
        g = self.nh // self.nkv
        s = f"{self.kind}-{c}-d{self.d}-B{self.B}-h{self.nh}g{g}"
        if self.kind == "self":
            s += f"-S{self.S}-kt{kt}" + ("-wg1empty" if self.S % 128 and self.S % 128 <= 64 else "")
            if self.seqlens is not None:
                s += "-pad" + "_".join(map(str, self.seqlens))
        elif self.kind == "cross":
            s += f"-S{self.S}-Skv{self.Skv}-kt{kt}"
        elif self.kind == "cache":
            s += f"-Sq{self.S}-past{self.Skv - self.S}" + ("-mask" if self.mask else "")
        else:
            s += f"-T{self.S}-lens" + "_".join(map(str, self.lens)) + f"-max{self.max_seqlen}"
        if self.scale is not None:
            s += f"-scale{self.scale}"
        if self.dist != "normal":
            s += f"-{self.dist}"
        return s + (f"-{self.tag}" if self.tag else "")


def _packed(lens, nh, nkv, d, causal, max_extra=0, **kw):
    return Case("packed", len(lens), sum(lens), nh, nkv, d, causal, lens=tuple(lens), max_seqlen=max(lens) + max_extra, **kw)


# S: 1 to 5 key tiles, the j + 2 ring refill (>= 3 tiles), an empty second warpgroup (S % 128 in 1..64), partial tiles
SELF_S = (1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 384, 577)
CASES = [Case("self", 2, S, 2, 2, d, causal) for d in (64, 128) for causal in (True, False) for S in SELF_S]
CASES += [
    # right padding: 0 (an all-padding entry), tile edges, and the full length
    Case("self", 9, 200, 2, 2, 128, True, seqlens=(0, 1, 63, 64, 65, 127, 128, 129, 200)),
    Case("self", 9, 200, 2, 1, 64, False, seqlens=(200, 129, 128, 127, 65, 64, 63, 1, 0)),
    # GQA groups 1, 2, 4, 8, nh
    Case("self", 1, 200, 8, 8, 128, True),
    Case("self", 2, 200, 8, 4, 64, True),
    Case("self", 1, 300, 32, 8, 128, True),
    Case("self", 1, 200, 32, 4, 64, False),
    Case("self", 1, 257, 32, 1, 128, True),
]
# cross (UNet attn2), non-causal, d = 64: kv rows are slices of one [B, Skv, 2 nkv d] buffer
CASES += [Case("cross", 1 if S == 4096 else 2, S, 2, 2, 64, Skv=Skv) for S in (64, 256, 1024, 4096) for Skv in (1, 77, 128, 129, 333)]
# kv-cache continuation: bottom-right causal mask, kv_rows > Skv with garbage past Skv, left-padded kv_mask on odd entries
CASES += [Case("cache", 2, Sq, 4, 2, 128 if i % 2 else 64, True, Skv=Sq + past, mask=True)
          for i, (Sq, past) in enumerate([(1, 0), (1, 127), (1, 128), (5, 123), (128, 128), (129, 200), (64, 1000)])]
CASES += [Case("cache", 2, 1, 4, 4, 128, True, Skv=128), Case("cache", 1, 129, 4, 1, 64, True, Skv=329)]
# packed: samples ending mid-tile, a zero-length sample, T % 64 != 0, max_seqlen above the longest sample
CASES += [
    _packed((100, 0, 129, 64, 37), 4, 2, 128, True, max_extra=71),
    _packed((100, 0, 129, 64, 37), 4, 2, 128, False, max_extra=71),
    _packed((1, 255, 128, 63, 0), 2, 2, 64, True, max_extra=1),
    _packed((190, 5, 300), 2, 1, 64, False),
]
# production sizes
CASES += [
    Case("self", 1, 2048, 32, 32, 128, True, tag="llm"),
    Case("self", 1, 4096, 5, 5, 64, False, tag="unet64"),
    Case("self", 1, 1024, 10, 10, 64, False, tag="unet32"),
    Case("self", 1, 1024, 20, 20, 64, False, tag="sdxl32"),
    Case("cross", 2, 4096, 5, 5, 64, Skv=77, tag="unet64"),
    Case("self", 1, 577, 16, 16, 64, False, tag="clip336"),
    Case("self", 2, 257, 16, 16, 64, False, tag="clip224"),
]
# non-default scale, sharp softmax, monotone row max
CASES += [
    Case("self", 2, 257, 2, 2, 64, True, scale=0.3),
    Case("self", 2, 200, 2, 2, 128, False, scale=0.3),
    Case("self", 2, 384, 2, 2, 128, True, dist="sharp"),
    Case("self", 2, 577, 2, 1, 64, False, dist="sharp"),
    Case("cross", 2, 1024, 2, 2, 64, Skv=333, dist="sharp"),
    Case("cache", 2, 64, 4, 2, 128, True, Skv=600, mask=True, dist="sharp"),
    Case("self", 2, 577, 2, 2, 64, False, dist="rise"),
    Case("self", 2, 384, 2, 2, 128, True, dist="rise"),
    Case("cross", 2, 256, 2, 2, 64, Skv=333, dist="rise"),
    Case("self", 2, 384, 2, 2, 64, True, dist="fall"),
    Case("self", 2, 577, 2, 2, 128, False, dist="fall"),
]
CASE_BY_ID = {c.id: c for c in CASES}
assert len(CASE_BY_ID) == len(CASES), "case ids must be unique"

GARBAGE = 3.0e4     # cache rows past Skv: large and finite


# ------------------------------------------------------------------------------------------------ inputs
def _g(seed):
    return torch.Generator().manual_seed(seed)


def _seed(case: Case, seed: int) -> int:
    return seed + sum(ord(ch) * (i + 1) for i, ch in enumerate(case.id)) % 1000003


def _shape_dist(case, x, is_k):
    """Apply the case's logit distribution to q [.., L, h, d] or k, in float32 before rounding."""
    if case.dist == "sharp":
        return x * math.sqrt(10.0)                     # q k^T / sqrt(d) with sd 10
    if case.dist in ("rise", "fall"):
        x = x.clone()
        if is_k:
            t = (torch.arange(x.shape[-3]) // 128).to(x.dtype)
            x[..., 0] = (3.0 if case.dist == "rise" else -3.0) * t[:, None]
        else:
            x[..., 0] = 8.0
    return x


def split_heads(buf, heads, d):
    """Views [..., n, d] of consecutive column blocks of a [..., cols] buffer, one per entry of `heads`, keeping the buffer's token
    stride on every axis (unflatten would renormalise the stride of a size-1 token axis, which the kernels read as the row pitch)."""
    views, col = [], 0
    for n in heads:
        views.append(buf.as_strided((*buf.shape[:-1], n, d), (*buf.stride()[:-1], d, 1), buf.storage_offset() + col))
        col += n * d
    return views


def make_inputs(case: Case, seed: int = 0, probe: str | None = None):
    """Seeded host inputs of one case, in the layout its entry takes.  dict with q [B, S, nh, d] / k, v (views), dout, and per kind:
    self/packed "qkv" (the fused buffer the views slice), cross "kv", cache "kc"/"vc" [B, kv_rows, nkv, d] and "mask" [B, mask_ld],
    self "seqlens", packed "cu".  probe: None (N(0, 1) inputs shaped by case.dist), "fwd" (q = 0, k / v / dout = +-1), "bwd_q" (q = 0,
    k / v / dout = +-1), "bwd_k" (k = 0, q / v / dout = +-1)."""
    B, S, nh, nkv, d = case.B, case.S, case.nh, case.nkv, case.d
    g = _g(_seed(case, seed) + {None: 0, "fwd": 1, "bwd_q": 2, "bwd_k": 3}[probe])

    def draw(*shape, is_k=None):
        if probe is not None:
            x = torch.randint(0, 2, shape, generator=g).float() * 2 - 1
            if (probe in ("fwd", "bwd_q") and is_k is False) or (probe == "bwd_k" and is_k is True):
                x.zero_()
            return x
        x = torch.randn(*shape, generator=g)
        return x if is_k is None else _shape_dist(case, x, is_k)

    lead = (S,) if case.kind == "packed" else (B, S)
    out = {}
    if case.kind in ("self", "packed"):
        qkv = torch.cat([draw(*lead, nh, d, is_k=False), draw(*lead, nkv, d, is_k=True), draw(*lead, nkv, d)], -2).to(BF)
        out["qkv"] = qkv.flatten(-2)
        out["q"], out["k"], out["v"] = split_heads(out["qkv"], (nh, nkv, nkv), d)
        if case.seqlens is not None:
            out["seqlens"] = torch.tensor(case.seqlens, dtype=torch.int32)
        if case.kind == "packed":
            out["cu"] = torch.tensor([0] + list(torch.tensor(case.lens).cumsum(0)), dtype=torch.int32)
    elif case.kind == "cross":
        out["q"] = draw(B, S, nh, d, is_k=False).to(BF)
        kv = torch.cat([draw(B, case.Skv, nkv, d, is_k=True), draw(B, case.Skv, nkv, d)], -2).to(BF)
        out["kv"] = kv.flatten(-2)
        out["k"], out["v"] = split_heads(out["kv"], (nkv, nkv), d)
    else:
        Skv = case.Skv
        rows = Skv + 40
        out["q"] = draw(B, S, nh, d, is_k=False).to(BF)
        kc = torch.empty(B, rows, nkv, d)
        vc = torch.empty(B, rows, nkv, d)
        kc[:, :Skv], vc[:, :Skv] = draw(B, Skv, nkv, d, is_k=True), draw(B, Skv, nkv, d)
        kc[:, Skv:] = GARBAGE * (torch.rand(B, rows - Skv, nkv, d, generator=g) * 2 - 1)
        vc[:, Skv:] = GARBAGE * (torch.rand(B, rows - Skv, nkv, d, generator=g) * 2 - 1)
        out["kc"], out["vc"] = kc.to(BF), vc.to(BF)
        out["k"], out["v"] = out["kc"][:, :Skv], out["vc"][:, :Skv]
        if case.mask:
            ld = (Skv + 63) // 64 * 64 + 64                    # wider than the kernel's minimum
            m = (torch.rand(B, ld, generator=g) < 0.5).to(torch.uint8)   # garbage past Skv: never read
            m[:, :Skv] = 1
            for b in range(1, B, 2):                            # left padding covering the first rows' every key
                m[b, :min(Skv, Skv - S + S // 2 + 1)] = 0
            out["mask"] = m
    out["dout"] = draw(*lead, nh * d).to(BF)
    return out


# ------------------------------------------------------------------------------------------------ a case as dense problems
def subproblems(case: Case, inp, device="cpu", fault=None):
    """[(rows, q, k, v, vis, qrow)]: the case as dense problems over which the restatements run; rows = slice of the packed sequence
    (packed: one problem per sample, as the kernel computes each sample alone) or None.  Faults as in `visibility`, plus "kv_tail"
    (the TMA zero fill past the last key visible: zero keys up to the end of its 128-key tile) and "packed_tail" (a packed sample's
    tile tail — the next sample's rows, then zero fill — visible as keys)."""
    dev = lambda t: t.to(device)  # noqa: E731
    if case.kind == "packed":
        T = case.S
        cu = [int(x) for x in inp["cu"]]
        pad = lambda t: torch.cat([t, torch.zeros(128, *t.shape[1:], dtype=t.dtype)])  # noqa: E731
        kp, vp = pad(inp["k"]), pad(inp["v"])
        res = []
        for b in range(case.B):
            r0, n = cu[b], cu[b + 1] - cu[b]
            if n == 0:
                continue
            nk = min(-(-n // 128) * 128, T - r0 + 128) if fault == "packed_tail" else n
            q = inp["q"][r0:r0 + n][None]
            k, v = kp[r0:r0 + nk][None], vp[r0:r0 + nk][None]
            vis, qrow = visibility(1, n, nk, case.causal, fault=fault if fault != "packed_tail" else None)
            if fault == "packed_tail" and case.causal:        # the tail sits past every row: the causal mask still hides it
                vis = vis & (torch.arange(nk)[None, None] <= torch.arange(n)[None, :, None])
            res.append((slice(r0, r0 + n), dev(q), dev(k), dev(v), vis.to(device), qrow.to(device)))
        return res
    q, k, v = inp["q"], inp["k"], inp["v"]
    B, S, Skv = case.B, case.S, case.keys
    vis, qrow = visibility(B, S, Skv, case.causal, seqlens=case.seqlens, kv_mask=inp.get("mask"), fault=fault)
    if fault == "kv_tail" and Skv % 128:
        ext = -(-Skv // 128) * 128
        z = torch.zeros(B, ext - Skv, *k.shape[2:], dtype=k.dtype)
        k, v = torch.cat([k, z], 1), torch.cat([v, z], 1)
        tail = qrow[:, :, None].expand(B, S, ext - Skv)
        if case.causal:
            tail = tail & (torch.arange(Skv, ext)[None, None] <= torch.arange(S)[None, :, None] + (Skv - S))
        vis = torch.cat([vis, tail], -1)
    return [(None, dev(q), dev(k), dev(v), vis.to(device), qrow.to(device))]


def _place(parts, full_shape, fill, axis):
    """Stitch per-sample results of a packed case along `axis` (the token axis) of a [1, ...] tensor."""
    dev, dt = parts[0][1].device, parts[0][1].dtype
    outp = torch.full(full_shape, fill, dtype=dt, device=dev)
    for rows, t in parts:
        idx = [slice(None)] * len(full_shape)
        idx[axis] = rows
        outp[tuple(idx)] = t
    return outp


def fwd_case(case: Case, inp, device="cpu", fault=None, dt=F64, rnd=True):
    """(pre, lse, mass) of the whole case: pre / mass [B, S, nh, d] (packed: [1, T, nh, d]), lse [B, nh, S] ([1, nh, T])."""
    hm = kv_head_map(case.nh, case.nkv, fault)
    subs = subproblems(case, inp, device, fault)
    res = [(rows, fwd_ref(q, k, v, vis, qrow, case.scale_v, kv_head=hm, dt=dt, rnd=rnd, fault=fault))
           for rows, q, k, v, vis, qrow in subs]
    if case.kind != "packed":
        return res[0][1]
    T, nh, d = case.S, case.nh, case.d
    pre = _place([(r, x[0]) for r, x in res], (1, T, nh, d), 0.0, 1)
    lse = _place([(r, x[1]) for r, x in res], (1, nh, T), INF, 2)
    mass = _place([(r, x[2]) for r, x in res], (1, T, nh, d), 0.0, 1)
    return pre, lse, mass


def bwd_case(case: Case, inp, o, lse, device="cpu", fault=None, dt=F64, rnd=True, dout=None):
    """((dq, dk, dv), (mass_dq, mass_dk, mass_dv)) of the whole case from the kernel's o [.., nh * d] and lse (the entry's layouts).
    Faults: those of `bwd_masks`, "gqa_mod" and "dkv_group" (dK / dV sum only the first group - 1 q heads of each kv head)."""
    nh, nkv, d = case.nh, case.nkv, case.d
    hm = kv_head_map(nh, nkv, fault)
    dkv_heads = None
    if fault == "dkv_group":
        dkv_heads = torch.arange(nh) % (nh // nkv) != nh // nkv - 1
    dout = inp["dout"] if dout is None else dout
    lead = (1, case.S) if case.kind == "packed" else (case.B, case.S)
    o4 = o.reshape(*lead, nh, d).to(device)
    do4 = dout.reshape(*lead, nh, d).to(device)
    lse3 = lse.reshape(lead[0], nh, case.S).to(device)
    res = []
    for rows, q, k, v, vis, qrow in subproblems(case, inp, device, fault):
        vdq, vkv = bwd_masks(vis, case.causal, fault)
        r = rows if rows is not None else slice(None)
        res.append((rows, bwd_ref(q, k, v, o4[:, r], lse3[:, :, r], do4[:, r], vdq, vkv, qrow, case.scale_v, kv_head=hm,
                                  dkv_heads=dkv_heads, dt=dt, rnd=rnd)))
    if case.kind != "packed":
        return res[0][1]
    T = case.S
    shapes = [(1, T, nh, d), (1, T, nkv, d), (1, T, nkv, d)]
    grads = tuple(_place([(r, x[0][i][0]) for r, x in res], shapes[i], 0.0, 1) for i in range(3))
    masses = tuple(_place([(r, x[1][i][0]) for r, x in res], shapes[i], 0.0, 1) for i in range(3))
    return grads, masses


def probe_fwd_case(case: Case, inp, device="cpu"):
    """Closed-form forward probe expectation (out, lse) of the whole case on probe inputs (make_inputs(probe="fwd"))."""
    hm = kv_head_map(case.nh, case.nkv)
    res = [(rows, probe_fwd_expect(v, vis, qrow, hm)) for rows, q, k, v, vis, qrow in subproblems(case, inp, device)]
    if case.kind != "packed":
        return res[0][1]
    T, nh, d = case.S, case.nh, case.d
    return (_place([(r, x[0][0]) for r, x in res], (1, T, nh, d), 0.0, 1),
            _place([(r, x[1][0]) for r, x in res], (1, nh, T), INF, 2))


def probe_bwd_case(case: Case, inp, device="cpu"):
    """Closed-form backward probe expectation (dq, dk, dv) on probe inputs (make_inputs(probe="bwd_q" / "bwd_k")), lse = 0, O = 0."""
    hm = kv_head_map(case.nh, case.nkv)
    do4 = inp["dout"].reshape(*((1, case.S) if case.kind == "packed" else (case.B, case.S)), case.nh, case.d).to(device)
    res = []
    for rows, q, k, v, vis, qrow in subproblems(case, inp, device):
        r = rows if rows is not None else slice(None)
        res.append((rows, probe_bwd_expect(q, k, v, do4[:, r], vis, vis, qrow, case.scale_v, hm)))
    if case.kind != "packed":
        return res[0][1]
    T, nh, nkv, d = case.S, case.nh, case.nkv, case.d
    shapes = [(1, T, nh, d), (1, T, nkv, d), (1, T, nkv, d)]
    return tuple(_place([(r, x[i][0]) for r, x in res], shapes[i], 0.0, 1) for i in range(3))

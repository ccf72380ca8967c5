"""The row kernels of every training step in float64, with componentwise error bounds derived from each kernel's order
of operations; shared by tests/test_norm_loss_reference_cpu.py and tests/test_norm_loss_reference_gpu.py.

Entry points (csrc/norm.cu, csrc/loss.cu, csrc/tokens.cu), restated from their operands as stored:
  layernorm_fwd       y = (x - mean) rstd gamma (eps 1e-5 inside the square root, variance over D), written to row
                      dest_row[m] (-1: not written); ycopy = bf16(y); xraw = bf16(x) (exact); stats = (mean, rstd).
                      fp16 y saturates at +-65504 (cvt.rn.satfinite): the clamp is applied to y64.
  layernorm_bwd(_det) dx = rstd (g - mean(g) - xh mean(g xh)) + dres + draw with g = gamma dy[src_row[m]] and
                      xh = (x - mean) rstd from the stored stats (src_row[m] = -1: dx = dres + draw); dx_bf16 = bf16(dx);
                      dgamma += sum over rows with a gradient of dy xh (NULL: not written).
  qk_l2norm_fwd/bwd   F.normalize times the scale: y = s x / max(|x|, 1e-12) over each 64-vector (h query heads, the
                      key), the value half of kv passed through; below the clamp the gradient is s dy / 1e-12 with no
                      projection term; dq_scale / dk_scale += sum dy xh (each may be NULL).
  cross_entropy(_det) dlogits = (softmax over the C real columns - onehot) grad_scale in bf16, zero for C <= c < Cp and
                      for ignored rows; loss_acc += (loss_scale sum of row losses, row count); _det: one (loss_scale
                      block sum, count) partial per block of 8 rows, added in block order.
  embed_scatter_add   dtable[src_row[m]] += scale dx[m] (src_row -1: nothing).

Error model.  u = 2^-23 per fp32 operation (gemm_reference.U), gamma(n) = n u / (1 - n u) for a chain of n
roundings; every bound is multiplied by SECOND_ORDER for the products of first-order terms, and a 16-bit store adds
half an ulp of its format at |value64| + bound (gemm_reference.half_ulp).

LayerNorm forward.  Lane sums of ((x + y) + z) + w per float4, then one add per chunk, then a 5-level butterfly: a term
passes at most k + 7 roundings (k = ceil(D / 128) chunks), the squares one more.  gemm_reference.ln_stats turns that
chain into (dmean, dvar), the IEEE divisions by D included; gemm_reference.ln_rstd adds the eps addition and rsqrtf's
2 ulp; gemm_reference.ln_y the three products of y.  The statistics are checked against the same bounds.

LayerNorm backward.  The kernel recomputes xh = fma(x, rstd, -mean rstd): the rounded -mean rstd gives
u |mean| rstd, the fma u |xh| -- a term the forward does not have, large when |mean| >> std.  g = gamma dy rounds (u).
s1 = sum g / D passes k + 8 roundings per term; s2 = sum g xh / D (two fma per chunk) 2k + 7, plus sum |g| dxh.
dx = fma(xh, -s2 rstd, fma(g, rstd, -s1 rstd)): the two rounded products and two fma add u each; dres and draw one add
each.  dgamma: each lane's fma chain over the rows of its warp (ceil(rows_per_block / WARPS)), WARPS warps, then the
blocks and the previous contents: gamma(n) (|dgamma0| + sum |dy xh|) + sum |dy| dxh with n the sum of the three
counts + 1.  The counts come from the launch (ln_bwd_launch restates launch_ln_bwd).

l2norm.  ss = sum of 64 squares: 8 fma per lane and 3 shuffle levels, gamma(11) relative (all terms positive); sqrtf
and the division are IEEE, so inv = 1 / max(sqrt(ss), eps) errs relatively by dinv = gamma(11) / 2 + 2u.  Forward
y = (x inv) s: dinv + 2u relative.  Backward xh = x inv (dinv + u), sg = dy s (u), dot = sum xh sg (gamma(11) and
the operand errors), o = (sg - xh dot) inv: two more roundings and inv's.  The scale sums chain the grid-stride
iterations of a thread, the 32 vector slots of a block, the blocks and the previous contents (qk_bwd_launch restates
qk_l2norm_bwd_impl's block cap).

Cross entropy.  The row max is exact.  __expf(a), a = x - mx rounded (u |a| relative on the result), errs by at most
2 + floor(1.173 |a|) ulp (CUDA intrinsic table) and flushes below 2^-126 (absolute floor).  se sums the 40 register
slots of a lane and 5 levels (gamma(45)); the streaming kernel (C or Cp > 1280) folds float4 groups into an online
(max, sum) per lane instead, which adds the rescaling factors' errors (see ce_ref); inv = grad_scale / se is IEEE.  g = v inv (u), minus grad_scale at the label
(u).  Row loss (mx + logf(se)) - x_label: dse / se, logf's 1 ulp and two additions.  A block adds its 8 row losses in
order (gamma(7)) and multiplies by loss_scale (u); blocks are added by fp32 atomics or in block order onto loss_acc's
contents (gamma(blocks + 1)).  The row count is exact.

Embedding scatter-add.  Each destination element receives its n products scale dx (rounded) by n fp32 additions in
some order (atomics) or in position order (_det): gamma(n + 1) (|dtable0| + sum |scale dx|).
"""
import torch

from gemm_reference import (FP16_MAX, SECOND_ORDER, U, fmt_of, gamma, half_ulp, ln_rstd, ln_stats, ln_y)  # noqa: F401

CE_MAX_C = 1280          # 32 lanes x kCeMaxPerLane: the register kernel's row limit (csrc/loss.cu)
CE_SLOTS = 40            # kCeMaxPerLane
QK_EPS = 1e-12


def store_bound(v64, e, dtype):
    """e plus half an ulp of the stored format at |v64| + e (none for fp32)."""
    if dtype == torch.float32:
        return e
    return e + half_ulp(v64.abs() + e, fmt_of(dtype))


def clamp16(v, dtype):
    return v.clamp(-FP16_MAX, FP16_MAX) if dtype == torch.float16 else v


# ------------------------------------------------------------------------------------------------ launch bookkeeping
def ln_nchunk(D):
    """The NCHUNK instantiation omlm_layernorm_fwd / _bwd dispatch to (1, 2, 4, 8 or 16)."""
    k = (D + 127) // 128
    return next(n for n in (1, 2, 4, 8, 16) if k <= n)


def ln_bwd_grid(D, sms):
    """(the most blocks launch_ln_bwd launches, WARPS): its per_sm blocks per SM, set by shared memory."""
    nc = ln_nchunk(D)
    warps = 8 if nc <= 8 else 4
    smem = warps * 2 * nc * 128 * 12 + nc * 128 * 4
    return sms * max(1, min(4, (220 * 1024) // smem)), warps


def ln_bwd_launch(M, D, sms):
    """(blocks, rows_per_block, WARPS) of launch_ln_bwd."""
    blocks, warps = ln_bwd_grid(D, sms)
    rpb = max((M + blocks - 1) // blocks, warps)
    return (M + rpb - 1) // rpb, rpb, warps


def qk_bwd_launch(M, h, sms):
    """(blocks, grid-stride iterations of a thread) of qk_l2norm_bwd_impl."""
    total = M * (h + 2)
    blocks = min((total + 31) // 32, sms * 8)
    return blocks, (total + blocks * 32 - 1) // (blocks * 32)


# ------------------------------------------------------------------------------------------------ LayerNorm
def ln_fwd_ref(x, g, y_dtype):
    """Float64 (y in source-row order, its bound, mean, rstd and their bounds) of layernorm_fwd on rows x [M, D]."""
    x, g = x.double(), g.double()
    D = x.shape[1]
    mean, var, dmean, dvar = ln_stats(x, ln_nchunk(D) + 8)
    y, e = ln_y(x, g, mean, var, dmean, dvar)
    rstd, drstd = ln_rstd(var, dvar)
    yc = clamp16(y, y_dtype)
    return dict(y=yc, y_bound=store_bound(yc, e, y_dtype), ycopy_bound=store_bound(y, e, torch.bfloat16), ycopy=y,
                mean=mean[:, 0], mean_bound=dmean[:, 0] * SECOND_ORDER, rstd=rstd[:, 0],
                rstd_bound=(rstd * drstd)[:, 0] * SECOND_ORDER)


def ln_bwd_ref(dy, x, stats, g, *, dres=None, draw=None, src_row=None, dgamma0=None, sms=132):
    """Float64 (dx, its bound, dx_bf16's bound, dgamma, its bound) of layernorm_bwd(_det).  dy [Mdy, D] bf16 (rows picked
    by src_row), x [M, D] fp32, stats [M, 2] fp32 as stored."""
    M, D = x.shape
    x, g = x.double(), g.double()
    mean, rstd = stats[:, 0:1].double(), stats[:, 1:2].double()
    if src_row is None:
        has = torch.ones(M, dtype=torch.bool, device=x.device)
        dyr = dy[:M].double()
    else:
        sr = src_row.long()
        has = sr >= 0
        dyr = dy.double()[sr.clamp_min(0)] * has[:, None]
    k = (D + 127) // 128
    gg = g * dyr
    xh = (x - mean) * rstd
    dxh = U * (mean.abs() * rstd + xh.abs())
    s1 = gg.mean(-1, keepdim=True)
    s2 = (gg * xh).mean(-1, keepdim=True)
    ds1 = gamma(k + 8) * gg.abs().mean(-1, keepdim=True) + U * s1.abs()
    ds2 = (gamma(2 * k + 7) * (gg * xh).abs().mean(-1, keepdim=True) + (gg.abs() * dxh).mean(-1, keepdim=True)
           + U * s2.abs())
    core = rstd * (gg - s1 - xh * s2)
    e = (rstd * (U * gg.abs() + ds1 + U * s1.abs() + xh.abs() * ds2 + U * (xh * s2).abs() + s2.abs() * dxh)
         + U * (rstd * (gg - s1)).abs() + U * core.abs())
    core = core * has[:, None]
    e = e * has[:, None]
    dx = core.clone()
    acc = core.abs()
    if dres is not None:
        dx = dx + dres.double()
        acc = acc + dres.double().abs()
        e = e + U * acc * has[:, None]             # 0 + dres is exact for rows without a gradient
    if draw is not None:
        dx = dx + draw.double()
        acc = acc + draw.double().abs()
        e = e + U * acc
    e = e * SECOND_ORDER
    out = dict(dx=dx, dx_bound=e, dx_bf16_bound=store_bound(dx, e, torch.bfloat16))
    blocks, rpb, warps = ln_bwd_launch(M, D, sms)
    n = (rpb + warps - 1) // warps + warps + blocks + 1
    prod = dyr * xh
    dg0 = dgamma0.double() if dgamma0 is not None else torch.zeros(D, dtype=torch.float64, device=x.device)
    out["dgamma"] = dg0 + prod.sum(0)
    out["dgamma_bound"] = (gamma(n) * (dg0.abs() + prod.abs().sum(0)) + (dyr.abs() * dxh).sum(0)) * SECOND_ORDER
    return out


# ------------------------------------------------------------------------------------------------ q/k l2norm
def _qk_vectors(q_raw, kv_raw, h):
    """(q vectors [M, h, 64], key vectors [M, 1, 64]) in float64."""
    M = q_raw.shape[0]
    return q_raw.double().view(M, h, 64), kv_raw.double()[:, :64].view(M, 1, 64)


DINV = gamma(11) / 2 + 2 * U


def _normalize(v):
    n = v.norm(dim=-1, keepdim=True)
    c = n.clamp_min(QK_EPS)
    return v / c, 1.0 / c, n < QK_EPS


def qk_fwd_ref(q_raw, kv_raw, q_scale, k_scale, h):
    """Float64 (qn [M, h*64], its bound, kvn [M, 128], its bound) of qk_l2norm_fwd (value half: exact copy)."""
    M = q_raw.shape[0]
    q, k = _qk_vectors(q_raw, kv_raw, h)
    outs = []
    for v, s in ((q, q_scale), (k, k_scale)):
        xh, _, _ = _normalize(v)
        y = xh * s.double()
        e = y.abs() * (DINV + 2 * U) * SECOND_ORDER
        outs.append((y.reshape(M, -1), store_bound(y, e, torch.bfloat16).reshape(M, -1)))
    (qn, qb), (kn, kb) = outs
    val = kv_raw.double()[:, 64:]
    return dict(qn=qn, qn_bound=qb, kvn=torch.cat([kn, val], 1), kvn_bound=torch.cat([kb, torch.zeros_like(val)], 1))


def qk_bwd_ref(dqn, dkvn, q_raw, kv_raw, q_scale, k_scale, h, *, dq_scale0=None, dk_scale0=None, sms=132):
    """Float64 (dq_raw, dkv_raw, their bounds, dq_scale, dk_scale, their bounds) of qk_l2norm_bwd(_det)."""
    M = q_raw.shape[0]
    q, k = _qk_vectors(q_raw, kv_raw, h)
    gq, gk = dqn.double().view(M, h, 64), dkvn.double()[:, :64].view(M, 1, 64)
    blocks, iters = qk_bwd_launch(M, h, sms)
    n = iters + 32 + blocks + 1
    res = {}
    for name, v, gv, s, ds0 in (("q", q, gq, q_scale, dq_scale0), ("k", k, gk, k_scale, dk_scale0)):
        xh, inv, clamped = _normalize(v)
        sg = gv * s.double()
        dot = (xh * sg).sum(-1, keepdim=True) * (~clamped)
        o = (sg - xh * dot) * inv
        dxh = xh.abs() * (DINV + U)
        ddot = (gamma(11) * (xh * sg).abs().sum(-1, keepdim=True) + (dxh * sg.abs()).sum(-1, keepdim=True)
                + U * (xh.abs() * sg.abs()).sum(-1, keepdim=True)) * (~clamped)
        e = (inv * (U * sg.abs() + dot.abs() * dxh + xh.abs() * ddot + U * (xh * dot).abs() + U * (sg - xh * dot).abs())
             + o.abs() * (DINV + U)) * SECOND_ORDER
        res[name] = (o.reshape(M, -1), store_bound(o, e, torch.bfloat16).reshape(M, -1))
        prod = (gv * xh).reshape(-1, 64)
        d0 = ds0.double() if ds0 is not None else torch.zeros(64, dtype=torch.float64, device=q.device)
        res["d" + name + "s"] = (d0 + prod.sum(0), (gamma(n) * (d0.abs() + prod.abs().sum(0))
                                                     + (gv.abs() * dxh).reshape(-1, 64).sum(0)) * SECOND_ORDER)
    val = dkvn.double()[:, 64:]
    return dict(dq=res["q"][0], dq_bound=res["q"][1],
                dkv=torch.cat([res["k"][0], val], 1),
                dkv_bound=torch.cat([res["k"][1], store_bound(val, torch.zeros_like(val), torch.bfloat16)], 1),
                dq_scale=res["dqs"][0], dq_scale_bound=res["dqs"][1], dk_scale=res["dks"][0], dk_scale_bound=res["dks"][1])


# ------------------------------------------------------------------------------------------------ cross entropy
def ce_labels(labels, rows, label_stride=1, rows_per_batch=0, batch_stride=0):
    """The label of each row as the kernels read it: labels[(r / rows_per_batch) * batch_stride + (r % rows_per_batch) *
    label_stride] from the flat storage starting at labels' first element (rows_per_batch = 0: one flat vector)."""
    if rows_per_batch <= 0:
        rows_per_batch, batch_stride = rows, 0
    r = torch.arange(rows, device=labels.device)
    idx = (r // rows_per_batch) * batch_stride + (r % rows_per_batch) * label_stride
    flat = labels.as_strided((int(idx.max()) + 1,), (1,))
    return flat[idx].long()


EXP_ULPS = 1.173         # __expf: at most 2 + floor(1.173 |x|) ulp


def ce_ref(logits, lab, C, Cp, *, grad_scale, loss_scale=1.0, ignore_index=-100, loss0=0.0):
    """Float64 (dlogits [rows, Cp], its bound, row losses, their bounds, kept-row mask, per-block partials of 8 rows and
    their bounds, the total, its bound, the row count) of cross_entropy(_det) with labels `lab` [rows]."""
    x = logits[:, :C].double()
    rows = x.shape[0]
    keep = lab != ignore_index
    safe = torch.where(keep, lab, torch.zeros_like(lab))
    mx = x.max(1, keepdim=True).values
    a = x - mx
    v = torch.exp(a)
    se = v.sum(1, keepdim=True)
    p = v / se
    dv = v * ((2 + torch.floor(EXP_ULPS * a.abs())) * U + U * a.abs()) + 2.0 ** -126
    if C > CE_MAX_C or Cp > CE_MAX_C:
        # ce_stream_kernel: a lane folds k float4 groups into its online (m, s), each fold rescaling s by
        # __expf(m - nm) (2 + floor(1.173 |m - nm|) ulp and a product; the |m - nm| of a lane add up to at most
        # mx - min x) and adding four terms; the lanes are rescaled once more to the row max and summed in 5 levels
        k = (C + 127) // 128 + 1
        xmin = x.min(1, keepdim=True).values
        dse = (gamma(5 * k + 16) + (3 * k + 3 + 2 * EXP_ULPS * (mx - xmin)) * U) * se + dv.sum(1, keepdim=True)
    else:
        dse = gamma(CE_SLOTS + 5) * se + dv.sum(1, keepdim=True)
    gs = abs(grad_scale)
    onehot = torch.zeros_like(x).scatter_(1, safe[:, None], 1.0)
    g = (p - onehot) * grad_scale
    e = (gs * (dv + p * dse) / se + 2 * U * gs * p + U * g.abs()) * SECOND_ORDER
    g, e = g * keep[:, None], e * keep[:, None]
    dl = torch.zeros(rows, Cp, dtype=torch.float64, device=x.device)
    eb = torch.zeros_like(dl)
    dl[:, :C], eb[:, :C] = g, store_bound(g, e, torch.bfloat16)
    lse = mx[:, 0] + torch.log(se[:, 0])
    xl = x.gather(1, safe[:, None])[:, 0]
    loss = (lse - xl) * keep
    lb = ((dse / se)[:, 0] + U * torch.log(se[:, 0]).abs() + U * (mx[:, 0].abs() + torch.log(se[:, 0]).abs())
          + U * loss.abs()) * keep * SECOND_ORDER
    nb = (rows + 7) // 8
    pad = nb * 8 - rows
    lp = torch.nn.functional.pad(loss, (0, pad)).view(nb, 8)
    lbp = torch.nn.functional.pad(lb, (0, pad)).view(nb, 8)
    part = lp.sum(1) * loss_scale
    part_b = (abs(loss_scale) * (lbp.sum(1) + gamma(7) * lp.abs().sum(1)) + U * part.abs()) * SECOND_ORDER
    total = loss0 + part.sum()
    total_b = part_b.sum() + gamma(nb + 1) * (abs(loss0) + part.abs().sum()) * SECOND_ORDER
    cnt = torch.nn.functional.pad(keep.double(), (0, pad)).view(nb, 8).sum(1)
    return dict(dlogits=dl, dlogits_bound=eb, loss=loss, loss_bound=lb, keep=keep, part=part, part_bound=part_b,
                part_count=cnt, total=float(total), total_bound=float(total_b), count=int(keep.sum()))


# ------------------------------------------------------------------------------------------------ embeddings
def scatter_ref(dtable0, src_row, dx, scale):
    """Float64 (dtable, its bound) of embed_scatter_add(_det)."""
    t = dtable0.double().clone()
    sr = src_row.long()
    ok = sr >= 0
    contrib = dx.double()[ok] * scale
    idx = sr[ok]
    t.index_add_(0, idx, contrib)
    absum = dtable0.double().abs().index_add(0, idx, contrib.abs())
    n = torch.zeros(t.shape[0], dtype=torch.float64, device=t.device).index_add_(0, idx, torch.ones_like(idx, dtype=torch.float64))
    g = torch.where(n > 0, (n + 1) * U / (1 - (n + 1) * U), torch.zeros_like(n))    # gamma(n + 1); untouched rows exact
    return t, g[:, None] * absum * SECOND_ORDER


# ------------------------------------------------------------------------------------------------ checks
def ratio(got, ref, bnd):
    """Worst |got - ref| / bnd (NaN in got counts as infinite; an exact match is 0 even where the bound is 0)."""
    err = (got.double() - ref.double()).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bnd.double().clamp_min(1e-300))
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    return float(r.max()) if r.numel() else 0.0


def check(got, ref, bnd, what):
    """Assert |got - ref| <= bnd everywhere and return the worst ratio; the message names the worst element."""
    err = (got.double() - ref.double()).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bnd.double().clamp_min(1e-300))
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    worst = float(r.max()) if r.numel() else 0.0
    if worst > 1.0:
        at = tuple(int(i) for i in torch.nonzero(r == r.max())[0])
        raise AssertionError(f"{what}: element {at} at {worst:.3g} x its bound (got {float(got[at]):.9g}, "
                             f"float64 {float(ref[at]):.9g}, bound {float(bnd[at]):.3g}); {int((r > 1).sum())} elements out")
    return worst


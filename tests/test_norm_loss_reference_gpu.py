"""LayerNorm, q/k l2norm, cross entropy and the embedding scatter-add on the H100 against float64, per element
(tests/norm_loss_reference.py: the restatements and their derived bounds).

Every output starts NaN-poisoned with sentinel rows past its end; rows a remap leaves unwritten must stay NaN and the
sentinels must survive.  A failure names the worst element in units of its bound.  The last test records the call forms
the engine issues in training, evaluation and generation, replays each against float64 and fails on any form the
explicit cases do not cover."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import call_forms  # noqa: E402
import norm_loss_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
SENT = 3.0
NAN = float("nan")


def _lib():
    from open_musiclm_b200 import lib
    return lib


def _sms():
    return _lib().num_sms()


WORST = {}      # output -> worst error / bound seen in this module (printed at its end; DESIGN.md section 4 quotes it)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst error / bound per output:", {k: round(v, 3) for k, v in sorted(WORST.items())})


def _chk(got, ref, bnd, what, family):
    r = R.check(got, ref, bnd, what)
    WORST[family] = max(WORST.get(family, 0.0), r)
    return r


def _poisoned(rows, cols, dtype, fill=NAN):
    """[rows + 2, cols] buffer: `fill` over the first rows, SENT in the two guard rows."""
    b = torch.full((rows + 2, cols), fill, device=DEV, dtype=dtype)
    b[rows:] = SENT
    return b


def _guards(buf, rows, what):
    assert bool((buf[rows:].float() == SENT).all()), f"{what}: guard rows written"


def _guarded_vec(n, fill):
    whole = torch.full((n + 64,), SENT, device=DEV)
    whole[32:32 + n] = fill
    return whole[32:32 + n], whole


def _vec_guards(whole, n, what):
    assert bool((whole[:32] == SENT).all()) and bool((whole[32 + n:] == SENT).all()), f"{what}: guard elements written"


# ------------------------------------------------------------------------------------------------ LayerNorm
LN_D = [4, 64, 124, 128, 132, 256, 260, 512, 516, 1024, 1028, 1536, 2048]
FWD_FORMS = [(yd, yc, xr, st, de) for yd in (BF16, F16) for yc in (0, 1) for xr in (0, 1) for st in (0, 1) for de in (0, 1)]
BWD_FORMS = [(det, dr, dw, sr, xb, ng) for det in (0, 1) for dr in (0, 1) for dw in (0, 1) for sr in (0, 1) for xb in (0, 1)
             for ng in (0, 1)]
FULL_M = (7, 513)                      # every form at these M; the other M take a rotating subset


def ln_m_values(D):
    """1, 7, 9, 513, the M at which the backward's rows_per_block is WARPS + 1, and the cfg2 size 16384."""
    blocks, warps = R.ln_bwd_grid(D, _sms())
    assert R.ln_bwd_launch(blocks * warps + 1, D, _sms())[1] == warps + 1
    return [1, 7, 9, 513, blocks * warps + 1, 16384]


def ln_forms(forms, M, D):
    if M in FULL_M:
        return list(forms)
    i = LN_D.index(D)
    return [forms[(i * 5 + j * 11 + M) % len(forms)] for j in range(3)]


def ln_key_fwd(D, f):
    return ("layernorm_fwd", R.ln_nchunk(D), str(f[0])) + tuple(f[1:])


def ln_key_bwd(D, f):
    return ("layernorm_bwd", R.ln_nchunk(D)) + tuple(f)


def explicit_ln_keys():
    return ({ln_key_fwd(D, f) for D in LN_D for f in FWD_FORMS} | {ln_key_bwd(D, f) for D in LN_D for f in BWD_FORMS})


def ln_inputs(M, D, seed, big_gamma=False):
    """Rows randn * 3 + 0.5 with exact-zero rows (pad rows), |mean| / std up to 1e3, a near-constant row (std 1e-3) and
    an outlier element; gamma ~ 1 with, optionally, a few 1e5 channels that drive fp16 y into saturation."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, D, device=DEV, generator=g) * 3 + 0.5
    if M > 1:
        x[1::7] = 0
    if M > 2:
        x[2] = 1e3 + torch.randn(D, device=DEV, generator=g)
    if M > 3:
        x[3] = 0.25 + 1e-3 * torch.randn(D, device=DEV, generator=g)
    if M > 4:
        x[4, D // 3] = 200.0
    if M > 5:
        x[5] = -300 + 3 * torch.randn(D, device=DEV, generator=g)
    gam = 1 + 0.3 * torch.randn(D, device=DEV, generator=g)
    if big_gamma:
        gam[D // 2:D // 2 + 4] = 1e5
    return x, gam


def ln_fwd_run(x, gam, form, dest=None):
    lib = _lib()
    M, D = x.shape
    yd, yc, xr, st, de = form
    y = _poisoned(M, D, yd)
    ycopy = _poisoned(M, D, BF16) if yc else None
    xraw = _poisoned(M, D, BF16) if xr else None
    stats = _poisoned(M, 2, F32) if st else None
    lib.layernorm_fwd(x, gam, y, xraw[:M] if xr else None, stats[:M] if st else None, dest if de else None,
                      ycopy=ycopy[:M] if yc else None)
    return y, ycopy, xraw, stats


def ln_fwd_check(x, gam, form, dest, what):
    M, D = x.shape
    y, ycopy, xraw, stats = ln_fwd_run(x, gam, form, dest)
    torch.cuda.synchronize()
    ref = R.ln_fwd_ref(x, gam, form[0])
    if form[4]:
        d = dest.long()
        src = torch.full((M,), -1, dtype=torch.long, device=DEV)
        src[d[d >= 0]] = torch.arange(M, device=DEV)[d >= 0]
    else:
        src = torch.arange(M, device=DEV)
    w = src >= 0
    s = src.clamp_min(0)
    for buf, key, bkey, fam in ((y, "y", "y_bound", "ln y " + str(form[0])), (ycopy, "ycopy", "ycopy_bound", "ln ycopy")):
        if buf is None:
            continue
        _guards(buf, M, what)
        _chk(buf[:M][w], ref[key][s][w], ref[bkey][s][w], f"{what} {key}", fam)
        assert bool(torch.isnan(buf[:M][~w].float()).all()), f"{what} {key}: rows no dest_row names were written"
    if xraw is not None:
        _guards(xraw, M, what)
        assert torch.equal(xraw[:M], x.to(BF16)), f"{what}: xraw"
    if stats is not None:
        _guards(stats, M, what)
        _chk(stats[:M, 0], ref["mean"], ref["mean_bound"], f"{what} mean", "ln mean")
        _chk(stats[:M, 1], ref["rstd"], ref["rstd_bound"], f"{what} rstd", "ln rstd")
    return ln_key_fwd(D, form)


def ln_bwd_check(x, gam, stats, dy, form, src_row, gen, what):
    lib = _lib()
    M, D = x.shape
    det, dr, dw, sr, xb, ng = form
    dres = torch.randn(M, D, device=DEV, generator=gen) if dr else None
    draw = torch.randn(M, D, device=DEV, generator=gen).to(BF16) if dw else None
    dx = _poisoned(M, D, F32)
    dxb = _poisoned(M, D, BF16) if xb else None
    dg0 = torch.randn(D, device=DEV, generator=gen)
    dg, whole = _guarded_vec(D, NAN if ng else 0.0)
    if not ng:
        dg.copy_(dg0)
    part = None
    if det:
        blocks = R.ln_bwd_launch(M, D, _sms())[0]
        part = torch.empty(blocks * D, device=DEV)
    lib.layernorm_bwd(dy, x, stats, gam, dx[:M], None if ng else dg, dres=dres, draw=draw, src_row=src_row if sr else None,
                      dx_bf16=dxb[:M] if xb else None, part=part)
    torch.cuda.synchronize()
    ref = R.ln_bwd_ref(dy, x, stats, gam, dres=dres, draw=draw, src_row=src_row if sr else None,
                       dgamma0=None if ng else dg0, sms=_sms())
    _guards(dx, M, what)
    _chk(dx[:M], ref["dx"], ref["dx_bound"], f"{what} dx", "ln dx")
    if xb:
        _guards(dxb, M, what)
        _chk(dxb[:M], ref["dx"], ref["dx_bf16_bound"], f"{what} dx_bf16", "ln dx_bf16")
    _vec_guards(whole, D, what)
    if ng:
        assert bool(torch.isnan(dg).all()), f"{what}: a NULL dgamma was written"
    else:
        _chk(dg, ref["dgamma"], ref["dgamma_bound"], f"{what} dgamma", "ln dgamma")
    return ln_key_bwd(D, form)


def _ln_cases():
    return [(D, j) for D in LN_D for j in range(6)]


@pytest.mark.parametrize("D,mi", _ln_cases(), ids=lambda v: str(v))
def test_layernorm_per_element(D, mi):
    M = ln_m_values(D)[mi]
    gen = torch.Generator(device=DEV).manual_seed(D * 100 + mi)
    perm = torch.randperm(M, device=DEV, generator=gen).to(torch.int32)
    dest = perm.clone()
    dest[::5] = -1                                        # rows whose output nobody reads
    for big in (False, True):
        x, gam = ln_inputs(M, D, D + M + big, big_gamma=big)
        for form in ln_forms(FWD_FORMS, M, D):
            if big and form[0] != F16:
                continue
            ln_fwd_check(x, gam, form, dest, f"ln fwd D={D} M={M} {form} big={big}")
    x, gam = ln_inputs(M, D, D + M)
    stats = torch.empty(M, 2, device=DEV)
    y = torch.empty(M, D, device=DEV, dtype=BF16)
    _lib().layernorm_fwd(x, gam, y, None, stats)
    dy = torch.randn(M, D, device=DEV, generator=gen).to(BF16)
    src = perm.clone()
    src[1::4] = -1                                        # rows without a gradient (positions no head reads)
    for form in ln_forms(BWD_FORMS, M, D):
        ln_bwd_check(x, gam, stats, dy, form, src, gen, f"ln bwd D={D} M={M} {form}")


def test_layernorm_det_is_repeatable_and_matches_default():
    lib = _lib()
    M, D = 4099, 1028
    x, gam = ln_inputs(M, D, 3)
    stats = torch.empty(M, 2, device=DEV)
    lib.layernorm_fwd(x, gam, torch.empty(M, D, device=DEV, dtype=BF16), None, stats)
    dy = torch.randn(M, D, device=DEV).to(BF16)
    outs = []
    for det in (True, True, False):
        dx, dg = torch.empty(M, D, device=DEV), torch.zeros(D, device=DEV)
        part = torch.empty(R.ln_bwd_launch(M, D, _sms())[0] * D, device=DEV) if det else None
        lib.layernorm_bwd(dy, x, stats, gam, dx, dg, part=part)
        outs.append((dx, dg))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[0][0], outs[2][0])                # dx does not depend on the dgamma reduction


# ------------------------------------------------------------------------------------------------ q/k l2norm
QK_H = [1, 2, 3, 8, 16]
QK_FORMS = [(det, nq, nk) for det in (0, 1) for nq in (0, 1) for nk in (0, 1)]


def qk_key_fwd(h):
    return ("qk_l2norm_fwd", h)


def qk_key_bwd(h, f):
    return ("qk_l2norm_bwd", h) + tuple(f)


def explicit_qk_keys():
    return {qk_key_fwd(h) for h in QK_H} | {qk_key_bwd(h, f) for h in QK_H for f in QK_FORMS}


def qk_m_values():
    """M (h + 2) not a multiple of 32 at every h; the larger M makes the backward's grid-stride loop iterate."""
    return [37, 2 * _sms() * 8 * 32 // 3 + 1]


def _qk_vectors(n, gen):
    """n bf16 64-vectors: random, exact zeros, norms 0.3e-12 and 0.8e-12 (below the clamp), large ones."""
    v = torch.randn(n, 64, device=DEV, generator=gen)
    v[1::9] = 0
    sub = v[2::9]
    v[2::9] = sub / sub.norm(dim=1, keepdim=True) * 0.3e-12
    sub = v[3::9]
    v[3::9] = sub / sub.norm(dim=1, keepdim=True) * 0.8e-12
    v[4::9] *= 1e3
    return v.to(BF16)


def qk_inputs(M, h, gen):
    q = _qk_vectors(M * h, gen).view(M, h * 64)
    kv = torch.cat([_qk_vectors(M, gen), torch.randn(M, 64, device=DEV, generator=gen).to(BF16)], 1).contiguous()
    qs = 0.5 + torch.rand(64, device=DEV, generator=gen)
    ks = 0.5 + torch.rand(64, device=DEV, generator=gen)
    dqn = torch.randn(M, h * 64, device=DEV, generator=gen)
    dkvn = torch.randn(M, 128, device=DEV, generator=gen)
    dqn.view(-1, 64)[5::9] = 0                            # zero upstream gradient (on random, zero and sub-eps vectors)
    dqn.view(-1, 64)[1::18] = 0
    dkvn[1::18, :64] = 0
    return q, kv, qs, ks, dqn, dkvn


def qk_fwd_check(q, kv, qs, ks, h, what):
    lib = _lib()
    M = q.shape[0]
    qn, kvn = _poisoned(M, h * 64, BF16), _poisoned(M, 128, BF16)
    lib.qk_l2norm_fwd(q, kv, qs, ks, qn, kvn, h)
    torch.cuda.synchronize()
    ref = R.qk_fwd_ref(q, kv, qs, ks, h)
    _guards(qn, M, what)
    _guards(kvn, M, what)
    _chk(qn[:M], ref["qn"], ref["qn_bound"], f"{what} qn", "qk qn")
    _chk(kvn[:M, :64], ref["kvn"][:, :64], ref["kvn_bound"][:, :64], f"{what} kn", "qk kn")
    assert torch.equal(kvn[:M, 64:], kv[:, 64:]), f"{what}: the value half is not passed through"
    return qk_key_fwd(h)


def qk_bwd_check(q, kv, qs, ks, dqn, dkvn, h, form, gen, what):
    lib = _lib()
    M = q.shape[0]
    det, nq, nk = form
    dq, dkv = _poisoned(M, h * 64, BF16), _poisoned(M, 128, BF16)
    q0, k0 = torch.randn(64, device=DEV, generator=gen), torch.randn(64, device=DEV, generator=gen)
    dqs, wq = _guarded_vec(64, NAN if nq else 0.0)
    dks, wk = _guarded_vec(64, NAN if nk else 0.0)
    if not nq:
        dqs.copy_(q0)
    if not nk:
        dks.copy_(k0)
    part = torch.empty(R.qk_bwd_launch(M, h, _sms())[0] * 128, device=DEV) if det else None
    lib.qk_l2norm_bwd(dqn, dkvn, q, kv, qs, ks, dq, dkv, None if nq else dqs, None if nk else dks, h, part=part)
    torch.cuda.synchronize()
    ref = R.qk_bwd_ref(dqn, dkvn, q, kv, qs, ks, h, dq_scale0=q0, dk_scale0=k0, sms=_sms())
    _guards(dq, M, what)
    _guards(dkv, M, what)
    _chk(dq[:M], ref["dq"], ref["dq_bound"], f"{what} dq_raw", "qk dq")
    _chk(dkv[:M, :64], ref["dkv"][:, :64], ref["dkv_bound"][:, :64], f"{what} dk_raw", "qk dk")
    assert torch.equal(dkv[:M, 64:], dkvn[:, 64:].to(BF16)), f"{what}: the value gradient is not passed through"
    _vec_guards(wq, 64, what)
    _vec_guards(wk, 64, what)
    for null, buf, key in ((nq, dqs, "dq_scale"), (nk, dks, "dk_scale")):
        if null:
            assert bool(torch.isnan(buf).all()), f"{what}: a NULL {key} was written"
        else:
            _chk(buf, ref[key], ref[key + "_bound"], f"{what} {key}", "qk " + key)
    return qk_key_bwd(h, form)


@pytest.mark.parametrize("mi", [0, 1])
@pytest.mark.parametrize("h", QK_H)
def test_qk_l2norm_per_element(h, mi):
    M = qk_m_values()[mi]
    gen = torch.Generator(device=DEV).manual_seed(h * 10 + mi)
    q, kv, qs, ks, dqn, dkvn = qk_inputs(M, h, gen)
    qk_fwd_check(q, kv, qs, ks, h, f"qk fwd h={h} M={M}")
    for form in QK_FORMS:
        qk_bwd_check(q, kv, qs, ks, dqn, dkvn, h, form, gen, f"qk bwd h={h} M={M} {form}")


def test_qk_l2norm_below_the_clamp_has_no_projection_term():
    """A vector of norm 0.8e-12 with a gradient along itself: F.normalize's gradient there is s dy / 1e-12 (the clamp's
    constant denominator); the projection (sg - xh (xh . sg)) / 1e-12 removes most of it."""
    lib = _lib()
    v = torch.zeros(1, 64, device=DEV)
    v[0, 0] = 0.8e-12
    q, kv = v.to(BF16), torch.cat([v, v], 1).to(BF16)
    one = torch.ones(64, device=DEV)
    dqn, dkvn = torch.zeros(1, 64, device=DEV), torch.zeros(1, 128, device=DEV)
    dqn[0, 0] = 1.0
    dq, dkv = torch.empty(1, 64, device=DEV, dtype=BF16), torch.empty(1, 128, device=DEV, dtype=BF16)
    lib.qk_l2norm_bwd(dqn, dkvn, q, kv, one, one, dq, dkv, None, None, 1)
    torch.cuda.synchronize()
    assert float(dq[0, 0]) == pytest.approx(float(torch.tensor(1e12, dtype=BF16)), rel=0), float(dq[0, 0])


# ------------------------------------------------------------------------------------------------ cross entropy
CE_C = [1, 2, 31, 32, 33, 101, 1025, 1279, 1280]
CE_PAD = ["none", "exact", "padded"]          # dlogits absent, Cp = C, Cp = C rounded up to 64


def ce_path(C, Cp):
    return "stream" if C > R.CE_MAX_C or Cp > R.CE_MAX_C else "register"


def ce_key(C, Cp, has_dl, det, strided):
    return ("cross_entropy", ce_path(C, Cp), has_dl, det, strided, has_dl and Cp > C)


def explicit_ce_keys():
    keys = set()
    for C in CE_C:
        for pad in CE_PAD:
            Cp = _ce_cp(C, pad)
            for det in (0, 1):
                for strided in (0, 1):
                    keys.add(ce_key(C, Cp, pad != "none", det, strided))
    return keys


def _ce_cp(C, pad):
    return C if pad in ("none", "exact") else (C + 63) // 64 * 64


def ce_inputs(C, width, rows, gen):
    """logits [rows, ld] with NaN past C (never read), labels 0, C - 1 and -100 at fixed rows, a dominant +1e4 logit,
    a row of equal logits (as test_codebooks_gpu._ce_case)."""
    x = torch.randn(rows, max(width, C), device=DEV, generator=gen) * 6
    x[:, C:] = NAN
    lab = torch.randint(0, C, (rows,), device=DEV, generator=gen, dtype=torch.int32)
    lab[0] = 0
    if rows > 1:
        lab[1] = C - 1
    if rows > 5:
        lab[4::5] = -100
    if rows > 2:
        x[2, min(17, C - 1)] = 1e4
    if rows > 3:
        x[3, :C] = 0.75
    return x, lab


def ce_check(x, lab_arg, lab, C, Cp, has_dl, det, what, view=None):
    """One call against float64: dlogits per element, the zero padding and ignored rows, the loss per block of 8 rows
    (det: its partials), the total and the exact row count."""
    lib = _lib()
    rows = x.shape[0]
    gs, ls, acc0 = 0.37, 0.5, 1.25
    dl = _poisoned(rows, Cp, BF16) if has_dl else None
    acc = torch.tensor([acc0, 2.0], device=DEV)
    nb = (rows + 7) // 8
    part = torch.full((2 * nb,), NAN, device=DEV) if det else None
    kw = view or {}
    lib.cross_entropy(x, lab_arg, C, acc, grad_scale=gs, dlogits=dl[:rows] if has_dl else None, loss_scale=ls, part=part, rows=rows, **kw)
    torch.cuda.synchronize()
    ref = R.ce_ref(x, lab, C, Cp, grad_scale=gs, loss_scale=ls, loss0=acc0)
    if has_dl:
        _guards(dl, rows, what)
        _chk(dl[:rows], ref["dlogits"], ref["dlogits_bound"], f"{what} dlogits", "ce dlogits " + ce_path(C, Cp))
        assert bool((dl[:rows, C:] == 0).all()) and bool((dl[:rows][~ref["keep"]] == 0).all()), f"{what}: padding / ignored rows"
    if det:
        p = part.view(nb, 2)
        _chk(p[:, 0], ref["part"], ref["part_bound"], f"{what} loss per block of 8 rows", "ce loss per block")
        assert torch.equal(p[:, 1].double(), ref["part_count"]), f"{what}: row count per block"
    got = torch.tensor([float(acc[0])], dtype=torch.float64)
    _chk(got, torch.tensor([ref["total"]], dtype=torch.float64), torch.tensor([ref["total_bound"]], dtype=torch.float64),
         f"{what} loss", "ce loss total")
    assert float(acc[1]) == 2.0 + ref["count"], f"{what}: row count {float(acc[1]) - 2} != {ref['count']}"


def token_logprob_check(rows, C, ld, lstride, rpb, bstride, gen, what):
    """token_logprob on logits [rows, ld] (NaN past C) with flat labels (rpb = 0) or the strided view, against the negated
    ce_ref row loss within its bound; 0 for labels outside [0, C); the rows past `rows` of out keep their sentinel.
    -> its coverage key ("token_logprob", strided)."""
    lib = _lib()
    x = torch.randn(rows, ld, device=DEV, generator=gen) * 3
    x[:, C:] = NAN
    if rpb:
        plane = torch.randint(0, C, ((rows // rpb + 1) * bstride + rpb * lstride,), device=DEV, generator=gen, dtype=torch.int32)
        plane[lstride] = -100
        plane[0] = C
        view = dict(label_stride=lstride, rows_per_batch=rpb, batch_stride=bstride)
        lab = R.ce_labels(plane, rows, **view)
    else:
        plane = torch.randint(0, C, (rows,), device=DEV, generator=gen, dtype=torch.int32)
        plane[::5] = -100
        plane[1::7] = C
        view, lab = dict(label_stride=lstride), plane.long()
    out = torch.full((rows + 2,), 7.0, device=DEV)
    lib.token_logprob(x, plane, C, out, rows=rows, **view)
    torch.cuda.synchronize()
    assert bool((out[rows:] == 7.0).all()), f"{what}: out written past its rows"
    lab = lab.to(DEV).long()
    valid = (lab >= 0) & (lab < C)
    ref = R.ce_ref(x, torch.where(valid, lab, torch.full_like(lab, -100)), C, C, grad_scale=0.0)
    got = out[:rows].double()
    assert bool((got[~valid] == 0).all()), f"{what}: labels outside [0, C) must give 0"
    err = (got + ref["loss"].to(DEV)).abs()[valid]
    bnd = ref["loss_bound"].to(DEV)[valid]
    assert bool((err <= bnd).all()), f"{what}: {int((err > bnd).sum())} rows beyond the bound, worst {float((err / bnd).max()):.3f}"
    WORST["token_logprob"] = max(WORST.get("token_logprob", 0.0), float((err / bnd).max()) if err.numel() else 0.0)
    return ("token_logprob", int(rpb > 0))


@pytest.mark.parametrize("pad", CE_PAD)
@pytest.mark.parametrize("C", CE_C)
def test_cross_entropy_register_path_per_element(C, pad):
    Cp = _ce_cp(C, pad)
    has_dl = pad != "none"
    gen = torch.Generator(device=DEV).manual_seed(C * 7 + len(pad))
    for rows in (1, 333, 8000 if C == 1025 else 20):
        x, lab = ce_inputs(C, Cp, rows, gen)
        for det in (0, 1):
            ce_check(x, lab, lab.long(), C, Cp, has_dl, det, f"ce C={C} Cp={Cp} rows={rows} det={det}")
    # the trainer's strided label view: rows ordered (sequence b, step t), labels at plane[b, off + qi + q t]
    B, cnt, q, qi, off = 9, 37, 3, 1, 5
    plane = torch.randint(0, C, (B, off + q * cnt + 2), device=DEV, dtype=torch.int32, generator=gen)
    plane[2, off + qi + q * 4] = -100
    x, _ = ce_inputs(C, Cp, B * cnt, gen)
    view = dict(label_stride=q, rows_per_batch=cnt, batch_stride=plane.stride(0))
    lab = R.ce_labels(plane[0, off + qi:], B * cnt, **view)
    for det in (0, 1):
        ce_check(x, plane[0, off + qi:], lab, C, Cp, has_dl, det, f"ce strided C={C} Cp={Cp} det={det}", view=view)


@pytest.mark.parametrize("C", [1, 1279, 1280])
def test_cross_entropy_dispatch_boundary_goes_to_the_streaming_kernel(C):
    """C <= 1280 with a gradient row wider than 1280 columns: the register kernel cannot write it; the streaming kernel
    must, with the same per-element bound."""
    Cp = 1344
    assert ce_path(C, Cp) == "stream"
    gen = torch.Generator(device=DEV).manual_seed(C)
    x = torch.randn(333, Cp, device=DEV, generator=gen) * 6
    x[:, C:] = NAN
    _, lab = ce_inputs(C, Cp, 333, gen)
    for det in (0, 1):
        ce_check(x, lab, lab.long(), C, Cp, True, det, f"ce boundary C={C} Cp={Cp} det={det}")


def test_cross_entropy_rejects_a_gradient_row_narrower_than_C():
    """A dlogits of rows x Cp with Cp < C would get a truncated gradient; both paths refuse it (the call itself stays in
    bounds: every kernel writes only below Cp)."""
    lib = _lib()
    for C in (101, 1025):
        x = torch.randn(16, C, device=DEV)
        lab = torch.zeros(16, device=DEV, dtype=torch.int32)
        acc = torch.zeros(2, device=DEV)
        with pytest.raises(lib.OmlmError, match="C <= Cp"):
            lib.cross_entropy(x, lab, C, acc, grad_scale=1.0, dlogits=torch.empty(16, C - 5, device=DEV, dtype=BF16))


# ------------------------------------------------------------------------------------------------ embeddings
@pytest.mark.parametrize("D", [64, 1032, 2048])
@pytest.mark.parametrize("det", [0, 1])
def test_embed_scatter_add_per_element(D, det):
    lib = _lib()
    gen = torch.Generator(device=DEV).manual_seed(D + det)
    rows, M = 50, 3001
    src = torch.randint(0, rows, (M,), device=DEV, generator=gen, dtype=torch.int32)
    src[::7] = -1
    src[100:400] = 3                                       # one row hit 300 times
    dx = torch.randn(M, D, device=DEV, generator=gen)
    t0 = torch.randn(rows, D, device=DEV, generator=gen)
    t = _poisoned(rows, D, F32, fill=0.0)
    t[:rows] = t0
    first = lib.embed_row_markers(rows, DEV) if det else None
    lib.embed_scatter_add(t[:rows], src, dx, 0.3, first=first)
    torch.cuda.synchronize()
    ref, bnd = R.scatter_ref(t0, src, dx, 0.3)
    _guards(t, rows, "scatter")
    _chk(t[:rows], ref, bnd, f"scatter D={D} det={det}", "embed_scatter_add")
    untouched = torch.ones(rows, dtype=torch.bool, device=DEV)
    untouched[src[src >= 0].long()] = False
    assert torch.equal(t[:rows][untouched], t0[untouched])
    if det:
        assert bool((first == 0x7FFFFFFF).all())
        again = t0.clone()
        lib.embed_scatter_add(again, src, dx, 0.3, first=first)
        assert torch.equal(again, t[:rows])


@pytest.mark.parametrize("two", [0, 1])
def test_embed_gather_exact(two):
    lib = _lib()
    gen = torch.Generator(device=DEV).manual_seed(two)
    table = torch.randn(40, 72, device=DEV, generator=gen)
    src = torch.randint(-1, 40, (301,), device=DEV, generator=gen, dtype=torch.int32)
    src2 = torch.randint(-1, 40, (301,), device=DEV, generator=gen, dtype=torch.int32) if two else None
    x = _poisoned(301, 72, F32)
    lib.embed_gather(table, src, x[:301], src2)
    torch.cuda.synchronize()
    want = table[src.long().clamp_min(0)] * (src >= 0)[:, None]
    if two:
        want = want + table[src2.long().clamp_min(0)] * (src2 >= 0)[:, None]
    assert torch.equal(x[:301], want)
    _guards(x, 301, "gather")


# ------------------------------------------------------------------------------------------------ the engine's call forms
NAMES = ("layernorm_fwd", "layernorm_bwd", "qk_l2norm_fwd", "qk_l2norm_bwd", "cross_entropy", "embed_gather", "embed_scatter_add",
         "token_logprob")


class _Recorder:
    """Wraps lib's row-kernel entry points (the engine and the trainer look them up as module attributes at call time)
    and records each call's form: shapes, formats and which optional operands are present."""

    def __init__(self, lib):
        self.lib, self.forms, self.phase, self.seen = lib, set(), None, set()
        self.orig = {n: getattr(lib, n) for n in NAMES}

    def _add(self, name, form):
        self.forms.add((name, form))
        self.seen.add((self.phase, name))

    def __enter__(self):
        o = self.orig

        def layernorm_fwd(x, gamma, y, xraw=None, stats=None, dest_row=None, ycopy=None):
            self._add("layernorm_fwd", (x.shape[0], x.shape[1], y.dtype, ycopy is not None, xraw is not None, stats is not None,
                                        dest_row is not None))
            return o["layernorm_fwd"](x, gamma, y, xraw, stats, dest_row, ycopy=ycopy)

        def layernorm_bwd(dy, x, stats, gamma, dx, dgamma, dres=None, draw=None, src_row=None, dx_bf16=None, part=None):
            self._add("layernorm_bwd", (x.shape[0], x.shape[1], part is not None, dres is not None, draw is not None,
                                        src_row is not None, dx_bf16 is not None, dgamma is None))
            return o["layernorm_bwd"](dy, x, stats, gamma, dx, dgamma, dres=dres, draw=draw, src_row=src_row, dx_bf16=dx_bf16, part=part)

        def qk_l2norm_fwd(q_raw, kv_raw, q_scale, k_scale, qn, kvn, heads):
            self._add("qk_l2norm_fwd", (q_raw.shape[0], heads))
            return o["qk_l2norm_fwd"](q_raw, kv_raw, q_scale, k_scale, qn, kvn, heads)

        def qk_l2norm_bwd(dqn, dkvn, q_raw, kv_raw, q_scale, k_scale, dq_raw, dkv_raw, dq_scale, dk_scale, heads, part=None):
            self._add("qk_l2norm_bwd", (q_raw.shape[0], heads, part is not None, dq_scale is None, dk_scale is None))
            return o["qk_l2norm_bwd"](dqn, dkvn, q_raw, kv_raw, q_scale, k_scale, dq_raw, dkv_raw, dq_scale, dk_scale, heads, part=part)

        def cross_entropy(logits, labels, C, loss_acc, *, grad_scale=0.0, dlogits=None, ignore_index=-100, label_stride=1, rows=None,
                          rows_per_batch=0, batch_stride=0, loss_scale=1.0, part=None):
            r = logits.shape[0] if rows is None else rows
            self._add("cross_entropy", (r, C, logits.stride(0), None if dlogits is None else dlogits.shape[1], part is not None,
                                        rows_per_batch > 0, label_stride, rows_per_batch, ignore_index))
            return o["cross_entropy"](logits, labels, C, loss_acc, grad_scale=grad_scale, dlogits=dlogits, ignore_index=ignore_index,
                                      label_stride=label_stride, rows=rows, rows_per_batch=rows_per_batch, batch_stride=batch_stride,
                                      loss_scale=loss_scale, part=part)

        def token_logprob(logits, labels, C, out, *, label_stride=1, rows=None, rows_per_batch=0, batch_stride=0):
            r = logits.shape[0] if rows is None else rows
            self._add("token_logprob", (r, C, logits.stride(0), label_stride, rows_per_batch, batch_stride))
            return o["token_logprob"](logits, labels, C, out, label_stride=label_stride, rows=rows, rows_per_batch=rows_per_batch,
                                      batch_stride=batch_stride)

        def embed_gather(table, src_row, x, src_row2=None):
            self._add("embed_gather", (src_row2 is not None,))          # (no device read here: generate captures graphs)
            return o["embed_gather"](table, src_row, x, src_row2)

        def embed_scatter_add(dtable, src_row, dx, scale, first=None):
            self._add("embed_scatter_add", (dx.shape[0], dx.shape[1], dtable.shape[0], first is not None))
            return o["embed_scatter_add"](dtable, src_row, dx, scale, first=first)

        for n in NAMES:
            setattr(self.lib, n, locals()[n])
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(self.lib, n, f)


def _record(act16, model, monkeypatch):
    """Forms of every phase of call_forms: default, deterministic, frozen-norm and frozen-relpos steps with pad tokens,
    eval_loss, generate and sessions."""
    with _Recorder(_lib()) as rec:
        call_forms.run(rec, model, act16, monkeypatch)
    # sessions: the packed prefill's final norm writes the rows dest_row names; return_logprobs scores the prefixes
    if model in call_forms.SONGS_ONLY:
        expected = {(p, n) for p in call_forms.SONG_PHASES for n in ("layernorm_fwd", "embed_gather")} | {("score songs", "token_logprob")}
    elif model in call_forms.BENCH_MODELS:
        expected = {(p, n) for p in ("bench step", "bench deterministic step") for n in NAMES if n not in ("embed_gather", "token_logprob")} | \
            {("bench step", "embed_gather"), ("eval_loss", "cross_entropy"), ("eval_loss", "layernorm_fwd")}
        if model in call_forms.GENERATION_MODELS:
            expected |= {("bench generation", "layernorm_fwd"), ("bench generation", "embed_gather")}
    else:
        expected = {(p, n) for p in call_forms.SESSION_PHASES for n in ("layernorm_fwd", "embed_gather")} | \
            {("session logprobs", "token_logprob"), ("session sampling", "token_logprob")}
    if model in call_forms.SCORE_MODELS:
        expected |= {("score", "layernorm_fwd"), ("score", "embed_gather"), ("score", "token_logprob")}
    if model in call_forms.MODELS and model not in call_forms.SESSIONS_ONLY:
        expected |= {(p, n) for p in ("default step", "deterministic step") for n in NAMES if n not in ("embed_gather", "token_logprob")} | \
            {("default step", "embed_gather"), ("eval_loss", "cross_entropy"), ("eval_loss", "layernorm_fwd"),
             ("generate B=3", "layernorm_fwd"), ("generate B=3", "embed_gather"), ("frozen norms step", "layernorm_bwd"),
             ("frozen norms step", "qk_l2norm_bwd")}
    assert expected <= rec.seen, f"entry points the engine did not call through lib: {sorted(expected - rec.seen)}"
    dest = {f[6] for n, f in rec.forms if n == "layernorm_fwd"}
    assert True in dest or model in call_forms.BENCH_MODELS, "no layernorm_fwd call with dest_row was recorded"
    return rec.forms


def _replay(name, f, gen):
    lib = _lib()
    if name == "layernorm_fwd":
        M, D, yd, yc, xr, st, de = f
        form = (yd, int(yc), int(xr), int(st), int(de))
        x, gam = ln_inputs(M, D, M + D, big_gamma=yd == F16)
        dest = torch.randperm(M, device=DEV, generator=gen).to(torch.int32)
        dest[::3] = -1
        return ln_fwd_check(x, gam, form, dest, f"engine form {name} {f}")
    if name == "layernorm_bwd":
        M, D, *flags = f
        form = tuple(int(v) for v in flags)
        x, gam = ln_inputs(M, D, M + D)
        stats = torch.empty(M, 2, device=DEV)
        lib.layernorm_fwd(x, gam, torch.empty(M, D, device=DEV, dtype=BF16), None, stats)
        dy = torch.randn(M, D, device=DEV, generator=gen).to(BF16)
        src = torch.randperm(M, device=DEV, generator=gen).to(torch.int32)
        src[::4] = -1
        return ln_bwd_check(x, gam, stats, dy, form, src, gen, f"engine form {name} {f}")
    if name == "qk_l2norm_fwd":
        M, h = f
        q, kv, qs, ks, _, _ = qk_inputs(M, h, gen)
        return qk_fwd_check(q, kv, qs, ks, h, f"engine form {name} {f}")
    if name == "qk_l2norm_bwd":
        M, h, det, nq, nk = f
        q, kv, qs, ks, dqn, dkvn = qk_inputs(M, h, gen)
        return qk_bwd_check(q, kv, qs, ks, dqn, dkvn, h, (int(det), int(nq), int(nk)), gen, f"engine form {name} {f}")
    if name == "cross_entropy":
        rows, C, ld, Cp, det, strided, lstride, rpb, ign = f
        assert ign == -100
        has_dl = Cp is not None
        Cp = Cp if has_dl else C
        x, lab = ce_inputs(C, ld, rows, gen)
        if strided:
            nb = rows // rpb
            plane = torch.randint(0, C, (nb, lstride * rpb + 3), device=DEV, dtype=torch.int32, generator=gen)
            plane[0, lstride * 2] = -100
            view = dict(label_stride=lstride, rows_per_batch=rpb, batch_stride=plane.stride(0))
            lab_arg, lab = plane[0], R.ce_labels(plane[0], rows, **view)
        else:
            view, lab_arg, lab = dict(label_stride=lstride), lab, lab.long()
        ce_check(x, lab_arg, lab, C, Cp, has_dl, int(det), f"engine form {name} {f}", view=view)
        return ce_key(C, Cp, has_dl, int(det), int(strided))
    if name == "token_logprob":
        rows, C, ld, lstride, rpb, bstride = f
        return token_logprob_check(rows, C, ld, lstride, rpb, bstride, gen, f"engine form {name} {f}")
    if name == "embed_gather":
        return ("embed_gather", int(f[0]))
    if name == "embed_scatter_add":
        return ("embed_scatter_add", int(f[3]))
    raise AssertionError(name)


@pytest.mark.parametrize("model", call_forms.MODEL_KEYS)
@pytest.mark.parametrize("act16", ["fp16", "bf16"])
def test_engine_call_forms_replayed_and_covered(act16, model, monkeypatch):
    forms = _record(act16, model, monkeypatch)
    gen = torch.Generator(device=DEV).manual_seed(23)
    covered = explicit_ln_keys() | explicit_qk_keys() | explicit_ce_keys()
    covered |= {("embed_gather", 0), ("embed_gather", 1)}               # test_embed_gather_exact
    covered |= {("embed_scatter_add", 0), ("embed_scatter_add", 1)}     # test_embed_scatter_add_per_element
    covered |= {("token_logprob", 0), ("token_logprob", 1)}             # test_logprobs_gpu: flat and strided labels
    keys = set()
    for name, f in sorted(forms, key=repr):
        keys.add(_replay(name, f, gen))
    print(f"act16={act16} {model}: {len(keys)} keys issued by the engine")
    for k in sorted(keys, key=repr):
        print("   ", k)
    missing = sorted((k for k in keys if k not in covered), key=repr)
    assert not missing, f"engine call forms without an explicit case: {missing}"

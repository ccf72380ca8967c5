"""The feed-forward middle against float64 (tests/ffn_reference.py), block by block and row by row at the seams.

Kernels: gemm_ffn_up (u = xn W1^T with the causal conv, GEGLU and the LayerNorm row sums in its epilogue), ffn_norm_fwd
(LayerNorm over F + dropout), ffn_mid_bwd in its default and fixed-order modes, and the row-sum epilogue of gemm_rowstat
that feeds it.  Forward activations are fp16 or bf16; gradients are bf16.

These kernels go wrong at seams: gemm_ffn_up emits 126-row tiles that overlap by two rows and resets the conv history at
sequence starts inside 16-row warp slabs; the backward walks 128-row tiles and recomputes two look-ahead rows per slab.
An error confined to one or two rows per tile hides in a tensor-wide norm, so every tensor gets
  (i)   componentwise: |got - ref| <= c 2^-p S, S the scale of ffn_reference.magnitude, 2^-p the unit of the stored
        format.  Derived, not measured; it catches local garbage.
  (ii)  the worst block error, ||got - ref|| / ||ref|| per (sequence, row tile, 128-channel group), row tiles of 126 rows
        (forward) or 128 rows (backward);
  (iii) the worst seam row: the same per (row, 128-channel group), over the first two rows of every sequence, the two
        rows on each side of every 126- and 128-row seam and the last two rows of every 16-row slab;
  (iv)  one rel-L2 over the tensor.
Each stage is compared twice where that tells errors apart: "iso" starts the reference from the kernel's own stored
upstream tensor (u, h, row sums), "chain" runs it from the original inputs.

BOUNDS (ii)-(iv) are about twice the worst value measured over every case of this file on an H100 80GB HBM3 (700 W
power limit); the measured worst values are listed beside them."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as nnf

pytestmark = pytest.mark.gpu
DEV = "cuda"
sys.path.insert(0, os.path.dirname(__file__))
import ffn_reference as FR  # noqa: E402

FLOOR = 0.1         # block norms below FLOOR x the RMS block norm of the reference count as FLOOR x RMS
GUARD = 3           # rows past M, filled with GUARD_VAL, that no kernel may touch
GUARD_VAL = 3.0
U32 = 2.0 ** -24
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
FLOOR_S = {torch.bfloat16: 0.0, torch.float16: 2.0 ** -14}       # ffn_reference.magnitude(floor=): fp16's subnormals

# (worst block, worst seam row, global rel-L2) per tensor.  Worst values measured over every case of this file on an
# H100 80GB HBM3 (700 W power limit), as (block, seam row, global):
#   u 2.2e-3 2.2e-3 1.7e-3             h iso 3.0e-3 3.2e-3 1.7e-3        h chain 6.8e-3 1.1e-2 3.1e-3
#   rowsum iso 4.2e-6 4.8e-6 1.5e-7    rowsum chain 4.9e-2 8.8e-2 2.5e-3 (sum_c h cancels; u's rounding stays)
#   stats iso 1.3e-7 1.7e-7 4.9e-8     stats chain 2.9e-3 3.5e-3 8.2e-4
#   hn iso 3.4e-3 3.6e-3 1.7e-3        hn chain 1.1e-2 1.7e-2 3.5e-3     LN-backward row sums 2.2e-6 2.7e-6 1.2e-6
#   du 9.7e-3 9.7e-3 1.8e-3 (the block and row figures at N = 1, where a block is one row)
#   dgamma 4.7e-7 - 4.4e-7             dconv_w 1.8e-3 - 1.2e-3
BOUNDS = {
    "u": (4.5e-3, 4.5e-3, 3.5e-3),
    "h iso": (6e-3, 6.5e-3, 3.5e-3),
    "h chain": (1.4e-2, 2.1e-2, 6.5e-3),
    "rowsum iso": (1e-5, 1e-5, 3e-7),
    "rowsum chain": (1e-1, 1.8e-1, 5e-3),
    "stats iso": (2.6e-7, 3.4e-7, 1e-7),
    "stats chain": (6e-3, 7e-3, 1.7e-3),
    "hn iso": (7e-3, 7.5e-3, 3.5e-3),
    "hn chain": (2.2e-2, 3.3e-2, 7e-3),
    "lnbwd sums": (4.4e-6, 5.5e-6, 2.4e-6),
    "du": (2e-2, 2e-2, 3.7e-3),
    "dgamma": (1e-6, 1e-6, 9e-7),
    "dconv_w": (3.7e-3, 3.7e-3, 2.4e-3),
}

# (d, F, conv, B, N): a* d = 72 (K tail 8) with a sequence start at every offset of the 126-row tile and 16-row slab;
# b* boundaries just before and on the tile seam; c an odd group count (no row-sum GEMM); d one real channel in the last
# group; e the plain FeedForward; f cfg2 width (352 persistent work items); g 40 row-sum partials per row; h cfg2 width with
# sequence starts on 16-row slab edges (224, 448) away from the 126-row seams
CASES = {
    "a1": (72, 192, True, 300, 1), "a2": (72, 192, True, 150, 2), "a3": (72, 192, True, 100, 3),
    "a127": (72, 192, True, 3, 127), "a129": (72, 192, True, 3, 129), "a252": (72, 192, True, 2, 252),
    "b125": (64, 170, True, 4, 125), "b126": (64, 170, True, 3, 126),
    "c": (128, 341, True, 2, 130),
    "d": (64, 129, True, 2, 200),
    "e": (72, 288, False, 3, 129),
    "f": (1024, 2730, True, 2, 1000),
    "g": (1280, 5120, False, 1, 300),
    "h": (1024, 2730, True, 3, 224),
}
ADT = {"bf16": torch.bfloat16, "fp16": torch.float16}


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as _lib
    _lib.device_check()
    return _lib


# ------------------------------------------------------------------------------------------------ metrics
def row_keys(B, N, fwd):
    """Block id of every row: (sequence, 126-row tile of the whole batch) forward, (sequence, 128-row tile) backward."""
    r = torch.arange(B * N, device=DEV)
    b, t = r // N, r % N
    tile = r // 126 if fwd else t // 128
    return b * (B * N // 126 + 2) + tile


def seam_rows(B, N):
    r = torch.arange(B * N, device=DEV)
    t, o6, o8 = r % N, r % 126, (r % N) % 128
    m = (t < 2) | (o6 < 2) | (o6 >= 124) | (o8 < 2) | (o8 >= 126) | (o6 % 16 >= 14) | (o8 % 16 >= 14) | (t >= N - 2)
    return m


def worst(x, ref, keys, cb):
    """x, ref [R, C]; a block is (the rows sharing a key) x (cb consecutive columns); rows with key < 0 are left out.
    -> (worst ||x - ref|| / max(||ref||, floor), (first row, column block)); floor = FLOOR x the RMS block norm of ref
    (1e-3 absolute where ref is all zero)."""
    x, ref = x.double(), ref.double()
    R, C = ref.shape
    nc = -(-C // cb)
    sel = keys >= 0
    _, inv = torch.unique(keys[sel], return_inverse=True)
    nb = int(inv.max()) + 1
    fold = lambda t: torch.zeros(nb, nc, dtype=torch.float64, device=t.device).index_add_(
        0, inv, nnf.pad(t[sel], (0, nc * cb - C)).view(-1, nc, cb).sum(-1))
    e2, r2 = fold((x - ref) ** 2), fold(ref ** 2)
    floor = FLOOR * float(r2.mean().sqrt()) or 1e-3
    err = e2.sqrt() / r2.sqrt().clamp_min(floor)
    k = int(err.argmax())
    first = int(torch.nonzero(sel)[(inv == k // nc).nonzero()[0, 0], 0])
    return float(err.flatten()[k]), (first, k % nc)


def check(fails, name, got, ref, allow, keys, seams, tag, cb=128):
    """Bounds (i)-(iv) of got against ref (2-D, rows = the keys' rows); violations are appended to fails."""
    got, ref = got.double(), ref.double()
    if not bool(torch.isfinite(got).all()):
        fails.append(f"{name} {tag}: non-finite values at {tuple(int(c) for c in (~torch.isfinite(got)).nonzero()[0])}")
        return
    err = (got - ref).abs()
    bad = err > allow
    ratio = float((err / allow.clamp_min(1e-300)).max())
    blk, at = worst(got, ref, keys, cb)
    row_keys_ = torch.where(seams, torch.arange(len(seams), device=DEV), torch.full_like(keys, -1))
    row, rat = worst(got, ref, row_keys_, cb) if bool(seams.any()) else (0.0, None)
    glob = float((got - ref).norm() / ref.norm().clamp_min(1e-30))
    b_blk, b_row, b_glob = BOUNDS[name]
    print(f"METRIC {name} {tag}: block {blk:.3e} at {at} (bound {b_blk:.1e}), seam row {row:.3e} at {rat} "
          f"(bound {b_row:.1e}), global {glob:.3e} (bound {b_glob:.1e}), componentwise {ratio:.3f} of the bound")
    if bool(bad.any()):
        idx = tuple(int(c) for c in bad.nonzero()[0])
        fails.append(f"{name} {tag}: {int(bad.sum())} entries beyond the componentwise bound, first at {idx}: got "
                     f"{float(got[idx]):.6e} ref {float(ref[idx]):.6e} allowed {float(allow[idx]):.3e}")
    if not blk < b_blk:
        fails.append(f"{name} {tag}: block at {at} error {blk:.3e} >= {b_blk:.1e}")
    if not row < b_row:
        fails.append(f"{name} {tag}: seam row {rat} error {row:.3e} >= {b_row:.1e}")
    if not glob < b_glob:
        fails.append(f"{name} {tag}: rel-L2 {glob:.3e} >= {b_glob:.1e}")


# ------------------------------------------------------------------------------------------------ reference rows
# The float64 references of forward_checks / backward_checks take about 1.3 GB per 1024 rows of F = 2730.  A form of more
# than REF_ROWS rows (bench.py's batches: 16384) is launched whole but compared sequence by sequence, on the first, a
# middle and the last: conv, GEGLU and LayerNorm never cross a sequence, so those rows' references are exact.  The
# weight gradients dgamma and dconv_w sum over every row; their references are accumulated over chunks of whole
# sequences of at most REF_ROWS rows.
REF_ROWS = 4096


def check_seqs(B, N):
    """The sequences a form is compared on: None (every row at once) up to REF_ROWS rows, else the first, a middle and
    the last."""
    return None if B * N <= REF_ROWS else sorted({0, B // 2, B - 1})


def row_groups(N, seqs, device=DEV):
    """Row indices of each reference group: [None] (every row) or one group per sequence of seqs."""
    if seqs is None:
        return [None]
    return [torch.arange(b * N, (b + 1) * N, device=device) for b in seqs]


def _sel(rows):
    return lambda t: t if (rows is None or t is None) else t[rows]


def _gtag(tag, rows, N):
    return tag if rows is None else f"{tag} sequence {int(rows[0]) // N}"


# ------------------------------------------------------------------------------------------------ set-up
def make_case(lib, key, adt, seed=0):
    """key: a name of CASES or a (d, F, conv, B, N) tuple."""
    d, F, use_conv, B, N = CASES[key] if isinstance(key, str) else key
    Fp, M = FR.padded(F), B * N
    g = torch.Generator(device=DEV).manual_seed(seed + F + N)
    xn = torch.randn(M, d, generator=g, device=DEV).to(adt)
    W1 = ((torch.rand(2 * F, d, generator=g, device=DEV) * 2 - 1) / math.sqrt(d)).to(adt)
    gam = 1 + 0.5 * torch.randn(F, generator=g, device=DEV)
    gam[F // 3] = -abs(float(gam[F // 3])) - 0.5                         # certainly some negative entries
    zero = sorted({0, F - 1, (2 * F) // 5} | ({127} if F > 127 else set()))
    gam[zero] = 0.0
    w1p = torch.empty(2 * Fp, d, device=DEV, dtype=adt)
    lib.pack(W1.float(), d, 2 * F, d, w1p, 2 * Fp, d, split_dst=-1, split_src=F)       # pack reads fp32
    if use_conv:
        cw = (torch.rand(2 * F, 3, generator=g, device=DEV) * 2 - 1) / math.sqrt(3)
        cwp = torch.empty(2 * Fp, 3, device=DEV)
        lib.pack(cw, 3, 2 * F, 3, cwp, 2 * Fp, 3, split_dst=-1, split_src=F)
    else:                       # FeedForward: taps pinned to (0, 0, 1), as the engine packs them
        cw = None
        cwp = torch.zeros(2 * Fp, 3, device=DEV)
        cwp[:, 2] = 1.0
    gp = torch.empty(Fp, device=DEV)
    lib.pack(gam, F, 1, F, gp, 1, Fp)
    return dict(d=d, F=F, Fp=Fp, B=B, N=N, M=M, xn=xn, W1=W1, w1p=w1p, cw=cw, cwp=cwp, gam=gam, gp=gp, zero=zero, adt=adt,
                g=g)


def guarded(rows, cols, dtype, fill=float("nan")):
    """[rows + GUARD, cols] filled with `fill`, guard rows GUARD_VAL -> (the whole buffer, its first `rows` rows)."""
    buf = torch.full((rows + GUARD, cols), fill, device=DEV, dtype=dtype)
    buf[rows:] = GUARD_VAL
    return buf, buf[:rows]


def guard_ok(fails, name, buf, rows):
    if not bool((buf[rows:] == GUARD_VAL).all()):
        fails.append(f"{name}: a guard row past M was written")




def run_up(lib, c, max_ctas):
    """gemm_ffn_up into NaN-poisoned, guarded outputs -> (u, h, rowsum) buffers with their guard rows."""
    M, Fp = c["M"], c["Fp"]
    ub, u = guarded(M, 2 * Fp, c["adt"])
    hb, h = guarded(M, Fp, c["adt"])
    rb, rs = guarded(M, Fp // 128 * 2, torch.float32)
    lib.gemm_ffn_up(c["xn"], c["w1p"], c["cwp"], u, h, rs, c["N"], Fp, max_ctas=max_ctas)
    return ub, hb, rb


def run_norm(lib, c, h, rs, p, copy=True):
    """ffn_norm_fwd -> (hn, the bf16 hn the backward reads, stats, keep bits or None, their guarded buffers).  fp16
    activations write the bf16 copy of hn (the training forward's form) unless copy is False (inference)."""
    M, F, Fp = c["M"], c["F"], c["Fp"]
    hnb, hn = guarded(M, Fp, c["adt"])
    sb, st = guarded(M, 2, torch.float32)
    f16 = c["adt"] == torch.float16 and copy
    hcb, hc = guarded(M, Fp, torch.bfloat16) if f16 else (hnb, hn)
    kb = torch.zeros(M + GUARD, Fp // 8, device=DEV, dtype=torch.uint8)
    kb[M:] = 0xA5
    seed = torch.tensor([1234 + Fp], dtype=torch.int64, device=DEV)
    lib.ffn_norm_fwd(h, rs, c["gp"], hn, st, F, Fp, p, seed, 3, keep_bits=kb[:M] if p > 0 else None,
                     hn_copy=hc if f16 else None)
    return dict(hn=hn, hn_b=hc, stats=st, kbits=kb[:M] if p > 0 else None, bufs=[hnb, sb, hcb], kb=kb)


def pad_cols(x, C):
    return nnf.pad(x, (0, C - x.shape[1]))


# ------------------------------------------------------------------------------------------------ forward
def norm_forms(adt):
    """(dropout p, bf16 copy of hn) of the forward checks: the training forms, and fp16 inference without the copy."""
    return [(p, True) for p in (0.0, 0.1, 0.5)] + ([(0.0, False)] if adt == torch.float16 else [])


@pytest.mark.parametrize("adt", list(ADT))
@pytest.mark.parametrize("key", list(CASES))
def test_forward_against_float64(lib, key, adt):
    c = make_case(lib, key, ADT[adt])
    fails = forward_checks(lib, c, f"{key} {adt}", (0, 1, 5), norm_forms(ADT[adt]))
    assert not fails, "\n".join(fails)


def forward_checks(lib, c, tag, max_ctas, norms, seqs=None):
    """gemm_ffn_up at each max_ctas (bit-identical to the first) and ffn_norm_fwd at each (p, copy) of norms, against
    float64 -> the list of failures.  seqs: the sequences whose rows are compared (None: every row; see REF_ROWS)."""
    F, Fp, B, N, M, unit = c["F"], c["Fp"], c["B"], c["N"], c["M"], UNIT[c["adt"]]
    fails = []
    runs = [run_up(lib, c, m) for m in max_ctas]
    torch.cuda.synchronize()
    ub, hb, rb = runs[0]
    for i, (u2, h2, r2) in enumerate(runs[1:]):
        for name, a, b in (("u", ub, u2), ("h", hb, h2), ("rowsum", rb, r2)):
            if not torch.equal(a, b):
                fails.append(f"{name}: max_ctas={max_ctas[i + 1]} differs from max_ctas={max_ctas[0]}")
    del runs[1:]
    for name, buf in (("u", ub), ("h", hb), ("rowsum", rb)):
        guard_ok(fails, name, buf, M)
    u, h, rs = ub[:M], hb[:M], rb[:M].view(M, Fp // 128, 2)
    if not bool((h[:, F:] == 0).all()):
        fails.append("h: padded columns are not zero")
    normed = []
    for p, copy in norms:
        ptag = f"p={p}{'' if copy else ' no copy'}"
        n = run_norm(lib, c, h, rs, p, copy)
        torch.cuda.synchronize()
        for name, buf in zip(("hn", "stats", "hn copy"), n["bufs"]):
            guard_ok(fails, name, buf, M)
        if not bool((n["kb"][M:] == 0xA5).all()):
            fails.append(f"keep bits {tag} {ptag}: a guard row past M was written")
        keep = None
        if p > 0:
            keep = FR.unpack_keep(n["kbits"], F)
            frac = 1 - float(keep.double().mean())
            if abs(frac - p) > 0.02:
                fails.append(f"dropout {tag} {ptag}: dropped fraction {frac:.4f}")
        if not bool((n["hn"][:, F:] == 0).all()):
            fails.append(f"hn {tag} {ptag}: padded columns are not zero")
        normed.append((p, copy, ptag, n, keep))
    keys_all, seams_all = row_keys(B, N, True), seam_rows(B, N)
    fl = FLOOR_S[c["adt"]]
    kern = lambda x: FR.to_kernel(x, F)
    for rows in row_groups(N, seqs):
        sel, gtag = _sel(rows), _gtag(tag, rows, N)
        keys, seams, xn, u_r, h_r, rs_r = sel(keys_all), sel(seams_all), sel(c["xn"]), sel(u), sel(h), sel(rs)
        chain = FR.forward(xn, c["W1"], c["cw"], c["gam"], N)
        Sc = FR.magnitude(xn, c["W1"], c["cw"], c["gam"], N, floor=fl)
        u_st = FR.from_kernel(u_r, F)
        iso = FR.forward(None, None, c["cw"], c["gam"], N, u=u_st)
        Si = FR.magnitude(None, None, c["cw"], c["gam"], N, u=u_st, floor=fl)
        # u: one rounding of an fp32 accumulation over d
        check(fails, "u", u_r, kern(chain["u"]), kern(2 * unit * Sc["u"]), keys, seams, gtag)
        # h: from the stored u (fp32 conv and GEGLU, one rounding) and from xn (plus u's rounding, through S_h)
        check(fails, "h iso", h_r, pad_cols(iso["h"], Fp), pad_cols(2 * unit * Si["h"], Fp), keys, seams, gtag)
        check(fails, "h chain", h_r, pad_cols(chain["h"], Fp), pad_cols(2 * unit * Sc["h"], Fp), keys, seams, gtag)
        # row sums of the unrounded fp32 h, added over the 128-channel tiles
        rsum = rs_r.double().sum(1)
        s_iso, s_chain = torch.stack([iso["s1"], iso["s2"]], 1), torch.stack([chain["s1"], chain["s2"]], 1)
        S_iso, S_chain = torch.stack([Si["s1"], Si["s2"]], 1), torch.stack([Sc["s1"], Sc["s2"]], 1)
        check(fails, "rowsum iso", rsum, s_iso, 2.0 ** -16 * S_iso, keys, seams, gtag, cb=1)
        check(fails, "rowsum chain", rsum, s_chain, 2 * unit * S_chain, keys, seams, gtag, cb=1)
        del iso, Si, s_iso, S_iso
        for p, copy, ptag, n, keep_all in normed:
            ptag = f"{gtag} {ptag}"
            keep, st = sel(keep_all), sel(n["stats"])
            # stats from the kernel's own row sums: fp32 E[h^2] - mean^2 and rsqrt
            mean_i = rsum[:, 0] / F
            var_i = (rsum[:, 1] / F - mean_i ** 2).clamp_min(0)
            rstd_i = (var_i + FR.EPS).rsqrt()
            a_abs = rs_r.double().abs().sum(1) / F
            allow_i = torch.stack([64 * U32 * a_abs[:, 0],
                                   64 * U32 * rstd_i ** 3 / 2 * (a_abs[:, 1] + mean_i ** 2) + 4 * U32 * rstd_i], 1)
            check(fails, "stats iso", st, torch.stack([mean_i, rstd_i], 1), allow_i, keys, seams, ptag, cb=1)
            allow_c = torch.stack([2 * unit * Sc["mean"] + 64 * U32 * Sc["mean"],
                                   2 * unit * Sc["rstd"] + 64 * U32 * Sc["rstd32"]], 1)
            check(fails, "stats chain", st, torch.stack([chain["mean"], chain["rstd"]], 1), allow_c, keys, seams, ptag, cb=1)
            # hn from the stored h and the kernel's stats (one rounding), and from xn
            r_iso = FR.forward(None, None, c["cw"], c["gam"], N, keep, p, u=u_st, h=h_r[:, :F], stats=(st[:, 0], st[:, 1]))
            S_hn_i = FR.magnitude(None, None, c["cw"], c["gam"], N, keep, p, u=u_st, floor=fl)["hn"]
            check(fails, "hn iso", sel(n["hn"]), pad_cols(r_iso["hn"], Fp), pad_cols(2 * unit * S_hn_i, Fp), keys, seams, ptag)
            if c["adt"] == torch.float16 and copy:
                check(fails, "hn iso", sel(n["hn_b"]), pad_cols(r_iso["hn"], Fp), pad_cols(2 * UNIT[torch.bfloat16] * S_hn_i, Fp),
                      keys, seams, ptag + " bf16 copy")
            del r_iso, S_hn_i
            r_ch = FR.forward(xn, c["W1"], c["cw"], c["gam"], N, keep, p)
            S_hn_c = FR.magnitude(xn, c["W1"], c["cw"], c["gam"], N, keep, p, floor=fl)["hn"]
            check(fails, "hn chain", sel(n["hn"]), pad_cols(r_ch["hn"], Fp), pad_cols((3 * unit + 64 * U32) * S_hn_c, Fp),
                  keys, seams, ptag)
            del r_ch, S_hn_c
        del chain, Sc
    return fails


# ------------------------------------------------------------------------------------------------ backward
def run_mid_bwd(lib, c, dhn, n, u, p, rowstat, parts, det, dg0, dc0):
    """ffn_mid_bwd into a NaN-poisoned, guarded du and onto the start values dg0 / dc0 -> (du buffer, dgamma, dconv_w)."""
    M, F, Fp, B, N = c["M"], c["F"], c["Fp"], c["B"], c["N"]
    dub, du = guarded(M, 2 * Fp, torch.bfloat16)
    dg = None if dg0 is None else dg0.clone()
    dc = None if dc0 is None else dc0.clone()
    part = None
    if det:
        part = torch.empty(B * ((N + 127) // 128) * 7 * F, device=DEV)
    lib.ffn_mid_bwd(dhn, n["hn_b"], u, n["stats"], c["cwp"], c["gp"], rowstat, du, dg, dc, B, N, F, Fp, p,
                    keep_bits=n["kbits"], rowstat_parts=parts, part=part)
    return dub, dg, dc


def check_grads(fails, c, dub, dg, dc, dg0, dc0, ref, S, tag, rows=None, weights=True):
    """du on `rows` (None: every row) against ref["du"] of those rows; with weights, dgamma and dconv_w (sums over
    every row) against ref's."""
    M, F, Fp, B, N = c["M"], c["F"], c["Fp"], c["B"], c["N"]
    sel = _sel(rows)
    guard_ok(fails, f"du {tag}", dub, M)
    du = sel(dub[:M])
    keys, seams = sel(row_keys(B, N, False)), sel(seam_rows(B, N))
    # du: one bf16 rounding; the row means m1, m2 inherit the bf16 hn (an error <= 2^-8 S_dh in dh)
    check(fails, "du", du, FR.to_kernel(ref["du"], F), FR.to_kernel(4 * 2.0 ** -8 * S["du"], F), keys, seams, tag)
    cols = FR.ileave_cols(F, DEV)[torch.tensor(c["zero"] + [F + z for z in c["zero"]], device=DEV)]
    r0 = ref["du"][:, torch.tensor(c["zero"] + [F + z for z in c["zero"]], device=DEV)]
    e0 = float((du[:, cols].double() - r0).norm() / r0.norm().clamp_min(1e-30))
    print(f"METRIC du at gamma = 0 {tag}: {e0:.3e}")
    if not e0 < BOUNDS["du"][0]:
        fails.append(f"du {tag}: rel-L2 {e0:.3e} at the channels whose gamma is 0")
    if not weights:
        return
    one = torch.zeros(1, dtype=torch.long, device=DEV)
    no = torch.zeros(1, dtype=torch.bool, device=DEV)
    if dg is not None:
        got = (dg.double() - dg0.double())[None]
        check(fails, "dgamma", got, ref["dgamma"][None], (2.0 ** -14 * S["dgamma"] + 2 * U32 * dg.double().abs())[None],
              one, no, tag)
    if dc0 is None:
        return
    taps = torch.arange(3, device=DEV)
    no3 = torch.zeros(3, dtype=torch.bool, device=DEV)
    got = FR.to_kernel((dc.double() - dc0.double()).t(), F)
    allow = FR.to_kernel((2.0 ** -8 * S["dconv_w"] + 2 * U32 * dc.double().abs()).t(), F)
    check(fails, "dconv_w", got, FR.to_kernel(ref["dconv_w"].t(), F), allow, taps, no3, tag)


def weight_grad_refs(c, u_st, dh, keep, p):
    """Float64 dgamma / dconv_w and their scales over every row, accumulated over chunks of whole sequences of at most
    REF_ROWS rows -> (ref, S) dicts."""
    F, N, B = c["F"], c["N"], c["B"]
    per = max(1, REF_ROWS // N)
    ref, S = {"dgamma": 0.0, "dconv_w": 0.0}, {"dgamma": 0.0, "dconv_w": 0.0}
    for b0 in range(0, B, per):
        rows = torch.arange(b0 * N, min(B, b0 + per) * N, device=u_st.device)
        sel = _sel(rows)
        r = FR.grads(sel(u_st), c["cw"], c["gam"], sel(dh)[:, :F], N, sel(keep), p)
        m = FR.magnitude(None, None, c["cw"], c["gam"], N, sel(keep), p, u=sel(u_st), dhn=sel(dh)[:, :F])
        for k in ("dgamma", "dconv_w"):
            if r[k] is not None:
                ref[k] = ref[k] + r[k]
                S[k] = S[k] + m[k]
        del r, m
    return ref, S


@pytest.mark.parametrize("adt", list(ADT))
@pytest.mark.parametrize("key", list(CASES))
def test_backward_against_float64(lib, key, adt):
    """ffn_mid_bwd against float64 autograd from the stored u, in its default and fixed-order modes, with the row sums
    from its own pass and (Fp % 256 == 0) from gemm_rowstat; gamma has exact zeros at channels 0, 127, F - 1 and one
    more.  dgamma and dconv_w accumulate onto non-zero start values.  Without dgamma (a frozen gamma): du and dconv_w
    against float64, in the fixed-order mode bit-identical to the call with it."""
    c = make_case(lib, key, ADT[adt])
    fails = backward_checks(lib, c, f"{key} {adt}", (0.0, 0.1, 0.5))
    assert not fails, "\n".join(fails)


def backward_checks(lib, c, tag, ps, dets=(False, True), max_ctas=0, seqs=None):
    """ffn_mid_bwd at each dropout p of ps and each mode of dets, with and without dgamma -> the list of failures.
    seqs: the sequences whose rows are compared (None: every row; see REF_ROWS)."""
    F, Fp, B, N, M, d = c["F"], c["Fp"], c["B"], c["N"], c["M"], c["d"]
    fails = []
    ub, hb, rb = run_up(lib, c, max_ctas)
    u, h, rs = ub[:M], hb[:M], rb[:M].view(M, Fp // 128, 2)
    u_st = FR.from_kernel(u, F)
    g = c["g"]
    dg0 = torch.randn(F, generator=g, device=DEV)
    dc0 = torch.randn(2 * F, 3, generator=g, device=DEV) if c["cw"] is not None else None
    groups = row_groups(N, seqs)
    for p in ps:
        n = run_norm(lib, c, h, rs, p)
        keep = None if p == 0 else FR.unpack_keep(n["kbits"], F)
        # d hn: a random bf16 gradient, and the product dx W2 of gemm_rowstat whose epilogue forms the row sums
        dhn = torch.zeros(M, Fp, device=DEV, dtype=torch.bfloat16)
        dhn[:, :F] = torch.randn(M, F, generator=g, device=DEV).bfloat16()
        variants = [("own", dhn, None)]
        if Fp % 256 == 0:
            dx = torch.randn(M, d, generator=g, device=DEV).bfloat16()
            w2 = ((torch.rand(d, Fp, generator=g, device=DEV) * 2 - 1) / math.sqrt(d)).bfloat16()
            w2[:, F:] = 0
            dhn2 = torch.empty(M, Fp, device=DEV, dtype=torch.bfloat16)
            pb, part = guarded(M, Fp // 128 * 2, torch.float32)
            ks = 1.0 / (1.0 - p) if p > 0 else 1.0
            lib.gemm_rowstat(dx, w2, dhn2, n["hn_b"], c["gp"], part, b_mn=True, M=M, N=Fp, K=d, keep_bits=n["kbits"],
                             keep_scale=ks)
            guard_ok(fails, "gemm_rowstat partials", pb, M)
            pv = part.view(M, Fp // 128, 2)
            for rows in groups:
                sel = _sel(rows)
                dxr, kr, hbr = sel(dx), sel(keep), sel(n["hn_b"])
                s1, s2 = FR.lnbwd_row_sums(dxr.double() @ w2.double(), hbr, c["gam"], kr, p)
                S1, S2 = FR.lnbwd_row_sums(dxr.double().abs() @ w2.double().abs(), hbr.double().abs(), c["gam"].abs(), kr, p)
                keys, seams = sel(row_keys(B, N, False)), sel(seam_rows(B, N))
                for j, (r, S) in enumerate(((s1, S1), (s2, S2))):
                    check(fails, "lnbwd sums", sel(pv)[..., j], r, 2.0 ** -16 * S, keys, seams,
                          f"{_gtag(tag, rows, N)} p={p} s{j + 1}", cb=Fp // 128)
                del s1, s2, S1, S2
            variants.append(("gemm", dhn2, part))
        for src, dh, part in variants:
            outs = []
            for det in dets:
                if part is None:
                    rowstat, parts = guarded(M, 2, torch.float32)[1], 0
                else:
                    rowstat, parts = part, Fp // 128
                dub, dg, dc = run_mid_bwd(lib, c, dh, n, u, p, rowstat, parts, det, dg0, dc0)
                torch.cuda.synchronize()
                dub2, _, dc2 = run_mid_bwd(lib, c, dh, n, u, p, rowstat, parts, det, None, dc0)
                torch.cuda.synchronize()
                if det and not (torch.equal(dub2, dub) and (dc is None or torch.equal(dc2, dc))):
                    fails.append(f"{tag} p={p} {src} det={det}: du / dconv_w without dgamma differ from the call with it")
                outs.append((det, dub, dg, dc, dub2, dc2))
            wref = weight_grad_refs(c, u_st, dh, keep, p) if seqs is not None else None
            for i, rows in enumerate(groups):
                sel = _sel(rows)
                ref = FR.grads(sel(u_st), c["cw"], c["gam"], sel(dh)[:, :F], N, sel(keep), p)
                S = FR.magnitude(None, None, c["cw"], c["gam"], N, sel(keep), p, u=sel(u_st), dhn=sel(dh)[:, :F])
                if wref is not None:
                    ref.update(wref[0])
                    S.update(wref[1])
                gtag = _gtag(tag, rows, N)
                for det, dub, dg, dc, dub2, dc2 in outs:
                    check_grads(fails, c, dub, dg, dc, dg0, dc0, ref, S, f"{gtag} p={p} {src} det={det}", rows, i == 0)
                    check_grads(fails, c, dub2, None, dc2, None, dc0, ref, S, f"{gtag} p={p} {src} det={det} dgamma=None",
                                rows, i == 0)
                del ref, S
    return fails

"""The 16-bit GEMMs (csrc/gemm_tc.cu) and the decode GEMMs (csrc/decode.cu skinny_gemm, csrc/decode_gemm.cu) in float64,
with a componentwise error bound derived from each kernel's accumulation structure; shared by
tests/test_gemm_reference_cpu.py and tests/test_gemm_reference_gpu.py.

Reference.  C64 = alpha * A B^T (+ addend, or + the output's previous contents) from the 16-bit operands as stored,
in the layout semantics of the entry point: operand majors, n_valid (columns >= n_valid are not written), and the
row remaps of the weight-gradient GEMMs:
  row_split > 0   source rows are halves of row_split rows; row r of half h goes to output row h * row_valid + r
                  when r < row_valid (the logit heads: row_split = Cp, row_valid = C), else nowhere;
  row_split < 0   the interleaved GEGLU order: source row 256 g + 128 s + c is channel ch = 128 g + c of the value
                  (s = 0) or gate (s = 1) half and goes to output row s * row_valid + ch when ch < row_valid.
decode_operand() restates the decode prologues: the 16-bit activation operand each one builds.

Error model.  Every product of two 16-bit values is exact in fp32 (bf16: 8 x 8 significant bits, fp16: 11 x 11).
Additions are the only error, and the tensor core is not assumed to round to nearest: a wgmma k16 step adds its 16
products and the accumulator after aligning them to the largest exponent, and may truncate.  With p = 24 significant
bits kept relative to the largest term, each of the 17 terms loses less than 2^-23 |largest| and the normalised sum
loses less than 2^-23 of itself, so one step errs by at most 18 u' sum|terms|, u' = 2^-23 (this also covers a
sequential chain of 16 truncating fp32 additions).  Over the T k16 steps of one split (T = 4 x the k-blocks the split
owns; zero-filled k tails add zero terms) the accumulator of step t is bounded by the absolute sum of every earlier
product, so
    |acc - sum_k a_k b_k| <= gamma(18 T) sum_k |a_k b_k|,       gamma(n) = n u' / (1 - n u').
Splits (atomic red.add onto the output's contents in any order, or gemm_splitk_det's partials added in split order)
are a chain of S more additions: gamma(S) (|out0| + sum|ab|).  The epilogue rounds acc * alpha (__fmul_rn) and then
adds the addend, u' (|alpha A B| + |addend|) between them (u' is twice the round-to-nearest unit: it absorbs the
second-order terms).  A bf16 store then rounds to nearest: half an ulp of the stored value.  Together

    |C - C64| <= (gamma_acc |alpha| (|A| |B|^T) + u' (|alpha A B| + |addend|) + gamma(S) |out0|) (1 + 2^-10)
                 + ulp_out(|C64| + that) / 2,

the factor 1 + 2^-10 covering the products of first-order terms (gamma <= 2^-10 for K <= 4104).  The decode GEMMs use
the same terms: decode_gemm runs the same wgmma steps over its K split and sums the splits in order (S - 1 additions);
skinny_gemm's lanes each chain ceil(K / 256) x 8 fmaf (exact products, one rounding each) before a 5-level warp sum.
The fp16 stores of the decode GEMMs clamp to +-65504 first; the clamp is applied to C64 here.

Prologue bound.  The prologue operand is y = (x - mean) rstd gamma (prologue 2: statistics of the fp32 row over K;
prologue 3: mean = s1 / n_real, var = max(s2 / n_real - mean^2, 0) from the row sums), rounded to the 16-bit format.
The fp32 statistics err by: the lane sums gamma(ceil(n / 32) + 6) of their absolute sums, the divisions u', the
variance additionally 2 |mean| dmean (+ dmean^2) and the cancellation u' (s2 / n + mean^2) of prologue 3; rstd then
errs relatively by dvar / (2 (var + eps)), half a unit for the eps addition and rsqrtf's 2 ulp (2^-22 relative).  The three fp32 products of y each round (3 u'), so

    |y32 - y| <= (|gamma| rstd (dmean + u' |x - mean|) + |y| (drstd + 3 u')) (1 + 2^-10)

and the 16-bit rounding adds half an ulp of the format at |y| + that.  Prologues 0 and 1 are exact up to that rounding.
"""
import math

import torch

U = 2.0 ** -23          # per-operation unit: covers truncation as well as round to nearest
EPS = 1e-5              # LayerNorm eps of both LayerNorm prologues
FP16_MAX = 65504.0
SECOND_ORDER = 1.0 + 2.0 ** -10
BK = 64                 # k-block of both wgmma kernels


def gamma(n, u=U):
    n = float(n)
    assert n * u < 0.5
    return n * u / (1.0 - n * u)


# ------------------------------------------------------------------------------------------------ split bookkeeping
def gemm_splits(K, splits):
    """(effective splits, k16 steps of the longest split): the host's clamp (gemm16_impl) -- every split owns a k-block."""
    kb = (K + BK - 1) // BK
    s = max(1, min(splits, kb))
    per = (kb + s - 1) // s
    return (kb + per - 1) // per, 4 * per


def gamma_gemm(K, splits=1):
    """gamma of the accumulator of omlm_gemm16 / gemm_splitk_det with `splits` (before the split sum)."""
    return gamma(18 * gemm_splits(K, splits)[1])


def gamma_skinny(K):
    return gamma(((K // 8 + 31) // 32) * 8 + 5)


# ------------------------------------------------------------------------------------------------ layouts
def operand(t, mn, rows, K):
    """Logical [rows, K] float64 view of a GEMM operand stored K-major ([rows, >= K]) or MN-major ([K, >= rows])."""
    return t[:K, :rows].t().double() if mn else t[:rows, :K].double()


def remap_sources(M, row_split=0, row_valid=0):
    """For each output row of a GEMM with this row remap, its source row (-1: no source row below M writes it)."""
    if row_split > 0:
        halves = (M + row_split - 1) // row_split
        h = torch.arange(halves).repeat_interleave(row_valid)
        r = torch.arange(row_valid).repeat(halves)
        src = h * row_split + r
    elif row_split < 0:
        ch = torch.arange(row_valid)
        base = (ch // 128) * 256 + ch % 128
        src = torch.cat([base, base + 128])
    else:
        src = torch.arange(M)
    return torch.where(src < M, src, torch.full_like(src, -1))


def ileave_cols(F):
    """The GEGLU remap as a gather: output row (value c | gate F + c) <- source row of the [., 2Fp] interleaved layout."""
    return remap_sources(2 * ((F + 127) // 128) * 128, -1, F)


def gemm_ref(a, b, *, a_mn=False, b_mn=False, M, N, K, alpha=1.0, addend=None, out0=None, row_split=0, row_valid=0, n_valid=0):
    """Float64 (C64, |A||B|^T, written) of one GEMM over its output rows (the remapped ones for row_split != 0) and its
    first n_valid columns.  addend: fp32 [rows, >= n_valid] added after alpha; out0: the output's contents before an
    accumulating call (split-K or gemm_splitk_det).  written: bool [rows] -- rows some source row maps to."""
    nv = n_valid if 0 < n_valid <= N else N
    A, B = operand(a, a_mn, M, K), operand(b, b_mn, N, K)
    prod = (A @ B[:nv].t()) * alpha
    absprod = (A.abs() @ B[:nv].abs().t()) * abs(alpha)
    src = remap_sources(M, row_split, row_valid).to(prod.device)
    written = src >= 0
    idx = src.clamp_min(0)
    prod = prod[idx] * written[:, None]
    absprod = absprod[idx] * written[:, None]
    c = prod.clone()
    if addend is not None:
        c += addend[:len(src), :nv].double()
    if out0 is not None:
        c += out0[:len(src), :nv].double()
    return c, absprod, written


def half_ulp(x, fmt):
    """Half an ulp of each |x| in fmt ('f32', 'bf16', 'f16'), with the format's subnormal spacing as the floor."""
    bits, emin = {"f32": (24, -126), "bf16": (8, -126), "f16": (11, -14)}[fmt]
    x = x.abs().double().clamp_min(2.0 ** emin)
    _, e = torch.frexp(x)                       # x = m 2^e, m in [0.5, 1): exact on every device (log2 / pow are not)
    return torch.ldexp(torch.ones_like(x), e - 1 - bits)


def fmt_of(dtype):
    return {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}[dtype]


def bound(c64, absprod, *, gamma_acc, out_dtype, addend=None, out0=None, gamma_split=0.0, alpha=1.0):
    """Componentwise bound of |C - C64| (see the module doc)."""
    e = gamma_acc * absprod + U * absprod                  # |alpha A B| <= |alpha| |A||B|^T
    if addend is not None:
        e = e + U * addend.double().abs()
    if out0 is not None:
        e = e + gamma_split * (out0.double().abs() + absprod)
    e = e * SECOND_ORDER
    return e + half_ulp(c64.abs() + e, fmt_of(out_dtype)) * (out_dtype != torch.float32)


# ------------------------------------------------------------------------------------------------ decode prologues
def round16(y, wdt):
    """Round float64 values to the 16-bit operand format as the kernels do (fp16: cvt.rn.satfinite saturates)."""
    if wdt == torch.float16:
        y = y.clamp(-FP16_MAX, FP16_MAX)
    return y.to(torch.float32).to(wdt).double()


def decode_operand(A, prologue, wdt, gamma_=None, rowsum=None, n_real=0, K=None):
    """(y64 before the 16-bit rounding, componentwise bound of the kernel's fp32 y against it) of the prologue's
    activation operand [B, K]; round16(y64) is the operand a correct kernel stores up to that bound."""
    K = A.shape[1] if K is None else K
    x = A[:, :K].double()
    if prologue in (0, 1):
        return x, torch.zeros_like(x)
    g = gamma_[:K].double()
    if prologue == 2:
        mean, var, dmean, dvar = ln_stats(x, math.ceil(K / 32) + 6)
    else:
        rs = rowsum.double()[:, :K // 128]
        s1, s2 = rs[..., 0].sum(-1, keepdim=True), rs[..., 1].sum(-1, keepdim=True)
        n = n_real
        mean = s1 / n
        var = (s2 / n - mean ** 2).clamp_min(0.0)
        ga = gamma(math.ceil(K / 128 / 32) + 6)
        dmean = ga * rs[..., 0].abs().sum(-1, keepdim=True) / n + U * mean.abs()
        ds2 = ga * rs[..., 1].abs().sum(-1, keepdim=True) / n + U * s2.abs() / n
        dvar = ds2 + 2 * mean.abs() * dmean + dmean ** 2 + 2 * U * (s2.abs() / n + mean ** 2)
    return ln_y(x, g, mean, var, dmean, dvar)


def ln_stats(x, chain):
    """Float64 (mean, var) of the rows of x, and the bounds (dmean, dvar) of fp32 statistics whose sums put each term
    through at most `chain` roundings (the square's product included) before the divisions by the row length."""
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    ga = gamma(chain)
    dmean = ga * x.abs().mean(-1, keepdim=True) + U * mean.abs()
    dvar = (ga * var + 2 * dmean * (x - mean).abs().mean(-1, keepdim=True) + dmean ** 2) * (1 + 2 * U) + U * var
    return mean, var, dmean, dvar


def ln_rstd(var, dvar):
    """Float64 rstd = 1 / sqrt(var + eps) and the relative bound of rsqrtf(var32 + eps) against it: the variance error,
    the rounding of the eps addition and rsqrtf's 2 ulp (at most 2^-22 relative)."""
    return 1.0 / torch.sqrt(var + EPS), dvar / (2 * (var + EPS)) + U / 2 + 2.0 ** -22


def ln_y(x, g, mean, var, dmean, dvar):
    """(y64 = (x - mean) rstd gamma, bound of the fp32 y = ((x - mean32) * rstd32) * gamma against it)."""
    rstd, drstd = ln_rstd(var, dvar)
    y = (x - mean) * rstd * g
    e = (g.abs() * rstd * (dmean + U * (x - mean).abs()) + y.abs() * (drstd + 3 * U)) * SECOND_ORDER
    return y, e


def operand_bound(y64, e32, wdt):
    """Bound of |stored 16-bit operand - y64|: the fp32 error and half an ulp of the format at |y| + e32."""
    return e32 + half_ulp(y64.abs() + e32, fmt_of(wdt))


def decode_ref(a_op, W, *, addend=None):
    """Float64 (C64, |A||W|^T) of a decode GEMM from its 16-bit activation operand a_op [B, K] and weights W [N, K]."""
    A, Wd = a_op.double(), W.double()
    c = A @ Wd.t()
    ab = A.abs() @ Wd.abs().t()
    if addend is not None:
        c = c + addend.double()
    return c, ab


def decode_bound(c64, absprod, *, K, out_dtype, gamma_acc, splits=1, addend=None):
    e = (gamma_acc + gamma(max(splits - 1, 0))) * absprod + U * absprod
    if addend is not None:
        e = e + U * addend.double().abs()
    e = e * SECOND_ORDER
    return e + half_ulp(c64.abs() + e, fmt_of(out_dtype)) * (out_dtype != torch.float32)


def clamp_out(c64, out_dtype):
    return c64.clamp(-FP16_MAX, FP16_MAX) if out_dtype == torch.float16 else c64


# ------------------------------------------------------------------------------------------------ reports
def worst(err, bnd, rows_blk=128, cols_blk=64):
    """(worst err / bound, its (row, col), the worst (rows_blk x cols_blk) block's index and its max ratio)."""
    err = err.double()
    r = torch.where(err == 0, torch.zeros_like(err), err / bnd.double().clamp_min(1e-300))
    r = torch.where(torch.isnan(r), torch.full_like(r, float("inf")), r)
    flat = int(r.argmax())
    i, j = divmod(flat, r.shape[1])
    R, Cn = r.shape
    pr, pc = (-R) % rows_blk, (-Cn) % cols_blk
    rp = torch.nn.functional.pad(r, (0, pc, 0, pr))
    blk = rp.reshape((R + pr) // rows_blk, rows_blk, (Cn + pc) // cols_blk, cols_blk).amax(dim=(1, 3))
    bflat = int(blk.argmax())
    bi, bj = divmod(bflat, blk.shape[1])
    return float(r[i, j]), (i, j), (bi, bj), float(blk[bi, bj])


def check(got, c64, bnd, what):
    """Assert |got - c64| <= bnd everywhere (NaN counts as a failure); return the worst ratio."""
    err = (got.double() - c64).abs()
    ratio, at, blk, blk_ratio = worst(err, bnd)
    assert ratio <= 1.0, (f"{what}: worst element {at} at {ratio:.3g} x its bound (got {float(got[at]):.9g}, "
                          f"float64 {float(c64[at]):.9g}); worst 128 x 64 block {blk} at {blk_ratio:.3g}")
    return ratio

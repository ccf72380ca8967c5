"""The 16-bit GEMMs (omlm_gemm16, gemm_splitk_det, gemm16_rowstat) and the decode GEMMs (skinny_gemm, decode_gemm)
against float64, per element, within the componentwise bounds derived in tests/gemm_reference.py.

Every output is NaN-poisoned before the call; the rows past M (or past the remapped rows), the columns past n_valid
and the pitch padding hold a sentinel that must survive.  A failure names the worst element in units of its bound and
the worst 128 x 64 block.  The persistent grid (max_ctas 1, 2, 7) must give bit-identical results for every form
without atomics, and the staged and direct epilogues bit-identical results at alpha = 1/3.  The engine's call forms
are recorded over the phases of tests/call_forms.py (training steps, generate and generation sessions) and replayed at their real shapes; a form whose coverage key the
explicit matrix below lacks fails the coverage test."""

import pytest
import torch

import call_forms
import gemm_reference as G

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = 3.0
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16

MAJORS = [(False, False), (False, True), (True, True)]
INSTS = [(a, b, bn, dt) for a, b in MAJORS for bn in (128, 256) for dt in (BF16, F16)]
M_VALS = [1, 63, 64, 65, 127, 129, 1000, 4100]
N_VALS = [8, 72, 136, 264, 1032]
K_VALS = [8, 56, 72, 520, 4104]


def r8(n):
    return (n + 7) // 8 * 8


def _lib():
    from open_musiclm_b200 import lib
    return lib


def _rand(shape, dt, gen, scale=1.0):
    return (torch.randn(shape, device=DEV, generator=gen) * scale).to(dt)


def _operand(rows, K, mn, dt, gen, strided):
    """A GEMM operand of logical shape [rows, K]: K-major [rows, ld >= K] or MN-major [K, ld >= rows], ld a multiple of 8
    (TMA's 16-byte pitches).  strided: ld grows by 8 and the operand is a row slice at row 5 of a larger buffer, as the
    engine takes its logit-head operands."""
    if mn:
        ld = r8(rows) + (8 if strided else 0)
        buf = _rand((K + (5 if strided else 0), ld), dt, gen)
    else:
        ld = K + (8 if strided else 0)
        buf = _rand((rows + (5 if strided else 0), ld), dt, gen)
    return buf[5:] if strided else buf


def _poisoned(rows, cols, ld, dt, extra_rows=2, fill=None):
    """[rows + extra_rows, ld] buffer: sentinel everywhere, NaN (or `fill`) over the [rows, cols] output region."""
    buf = torch.full((rows + extra_rows, ld), SENT, device=DEV, dtype=dt)
    buf[:rows, :cols] = float("nan") if fill is None else fill
    return buf


WORST = {}      # family -> worst error / bound seen in this module (printed at its end; DESIGN.md section 4 quotes it)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for fam in sorted(WORST):
        print(f"worst error / bound  {fam:28s} {WORST[fam]:.3f}")


def _note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    return ratio


def _guards_intact(buf, rows, cols, what):
    mask = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
    mask[:rows, :cols] = False
    bad = buf[mask] != SENT
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} guard elements written (rows past the output, columns past n_valid, pitch)"


def _gemm_check(got, c64, ab, *, K, splits=1, out_dtype, addend=None, out0=None, what, family="gemm16"):
    s, _ = G.gemm_splits(K, splits)
    bnd = G.bound(c64, ab, gamma_acc=G.gamma_gemm(K, splits), out_dtype=out_dtype, addend=addend, out0=out0,
                  gamma_split=G.gamma(s) if out0 is not None else 0.0)
    return _note(f"{family} {'fp32' if out_dtype == F32 else 'bf16'} out", G.check(got, c64, bnd, what))


# ------------------------------------------------------------------------------------------------ coverage keys
def staged_path(*, out_dtype, ldo, out_ptr, addend_ld=None, addend_ptr=None, atomic, row_split, n_valid):
    """gemm16_impl's choice of the staged (TMA) epilogue."""
    esz = 4 if out_dtype == F32 else 2
    vec_ok = (ldo * esz) % 16 == 0 and out_ptr % 16 == 0 and (addend_ld is None or ((addend_ld * 4) % 16 == 0 and addend_ptr % 16 == 0))
    return (not atomic and row_split == 0 and vec_ok and (addend_ld is None or out_dtype == F32) and (n_valid * esz) % 16 == 0)


def gemm_key(*, dt, a_mn, b_mn, block_n, out_dtype, addend, atomic, row_split, nv_short, staged):
    return ("gemm", str(dt), bool(a_mn), bool(b_mn), block_n, str(out_dtype), addend, bool(atomic),
            (row_split > 0) - (row_split < 0), bool(nv_short), bool(staged))


def explicit_gemm_keys():
    """Keys of every omlm_gemm16 form the tests below issue (kept next to them: a new form needs a new case)."""
    keys = set()
    for a_mn, b_mn, bn, dt in INSTS:
        k = dict(dt=dt, a_mn=a_mn, b_mn=b_mn, block_n=bn)
        for od in (BF16, F32):
            for staged in (True, False):
                keys.add(gemm_key(**k, out_dtype=od, addend="none", atomic=False, row_split=0, nv_short=False, staged=staged))
                keys.add(gemm_key(**k, out_dtype=od, addend="none", atomic=False, row_split=0, nv_short=True, staged=staged))
        for staged in (True, False):
            for nv_short in (False, True):
                keys.add(gemm_key(**k, out_dtype=F32, addend="separate", atomic=False, row_split=0, nv_short=nv_short, staged=staged))
                keys.add(gemm_key(**k, out_dtype=F32, addend="in_place", atomic=False, row_split=0, nv_short=nv_short, staged=staged))
        for nv_short in (False, True):
            keys.add(gemm_key(**k, out_dtype=F32, addend="none", atomic=True, row_split=0, nv_short=nv_short, staged=False))
    for sign, bn, dt, form, nv_short in REMAP_CASES_KEYS():
        keys.add(gemm_key(dt=dt, a_mn=True, b_mn=True, block_n=bn, out_dtype=F32, addend="in_place" if form == "in_place" else "none",
                          atomic=form == "atomic", row_split=sign, nv_short=nv_short, staged=False))
    return keys


# ------------------------------------------------------------------------------------------------ omlm_gemm16: the matrix
def _shapes(idx):
    """Eight (M, N, K) per instantiation: every M, N and K value with every instantiation, different pairings each."""
    return [(M_VALS[i], N_VALS[(i + idx) % 5], K_VALS[(2 * i + idx) % 5]) for i in range(8)]


CASES = [(inst, shape, j % 2 == 1) for idx, inst in enumerate(INSTS) for j, shape in enumerate(_shapes(idx))]


def _ids(c):
    (a_mn, b_mn, bn, dt), (M, N, K), strided = c
    return f"{'mn' if a_mn else 'k'}{'mn' if b_mn else 'k'}-bn{bn}-{'f16' if dt == F16 else 'bf16'}-{M}x{N}x{K}{'-strided' if strided else ''}"


def _grid_invariant(run, buf, what):
    """run(max_ctas) re-initialises buf's output region and calls; max_ctas 1, 2, 7 must give the default grid's bits."""
    ref = buf.clone()
    for mc in (1, 2, 7):
        run(mc)
        torch.cuda.synchronize()
        assert torch.equal(buf, ref), f"{what}: max_ctas={mc} differs from the default grid"


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_gemm16_per_element(case):
    lib = _lib()
    (a_mn, b_mn, bn, dt), (M, N, K), strided = case
    gen = torch.Generator(device=DEV).manual_seed(M * 131 + N * 7 + K + bn)
    a, b = _operand(M, K, a_mn, dt, gen, strided), _operand(N, K, b_mn, dt, gen, strided)
    kw = dict(a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, block_n=bn)
    c64, ab, _ = G.gemm_ref(a, b, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K)
    tag = _ids(case)
    # plain stores, bf16 and fp32, staged (16-byte pitch) and direct (odd pitch), full width and two n_valid tails
    for od in (BF16, F32):
        nvs = [N] + ([N - 8] if N > 8 else []) + ([N - 3] if N > 3 else [])
        for nv in nvs:
            outs = []
            for ldo in (r8(N) + 8, N + 1):
                buf = _poisoned(M, nv, ldo, od)

                def run(mc=0):
                    buf[:M, :nv] = float("nan")
                    lib.gemm(a, b, buf, n_valid=nv if nv < N else 0, max_ctas=mc, **kw)
                run()
                torch.cuda.synchronize()
                what = f"{tag} out={od} ldo={ldo} n_valid={nv}"
                _gemm_check(buf[:M, :nv], c64[:, :nv], ab[:, :nv], K=K, out_dtype=od, what=what)
                _guards_intact(buf, M, nv, what)
                _grid_invariant(run, buf, what)
                outs.append(buf[:M, :nv])
            assert torch.equal(outs[0], outs[1]), f"{tag} out={od} n_valid={nv}: staged and direct epilogues differ"
    # fp32 with the addend at alpha = 1/3: out of place and in place, staged and direct -- bit-identical
    X = torch.randn(M, N, device=DEV, generator=gen) * 4
    c3, ab3, _ = G.gemm_ref(a, b, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, alpha=1 / 3, addend=X)
    res = {}
    for ldo in (r8(N) + 8, N + 1):
        for form in ("separate", "in_place"):
            buf = _poisoned(M, N, ldo, F32)
            add = _poisoned(M, N, ldo, F32, fill=0.0)
            add[:M, :N] = X
            if form == "in_place":
                add = buf

            def run(mc=0):
                buf[:M, :N] = X if form == "in_place" else float("nan")
                lib.gemm(a, b, buf, addend=add, alpha=1 / 3, max_ctas=mc, **kw)
            run()
            torch.cuda.synchronize()
            what = f"{tag} addend={form} ldo={ldo} alpha=1/3"
            _gemm_check(buf[:M, :N], c3, ab3, K=K, out_dtype=F32, addend=X, what=what)
            _guards_intact(buf, M, N, what)
            _grid_invariant(run, buf, what)
            res[(ldo, form)] = buf[:M, :N].clone()
    vals = list(res.values())
    assert all(torch.equal(vals[0], v) for v in vals[1:]), f"{tag}: staged / direct / in-place results differ at alpha = 1/3"
    # the fp32 forms of a weight gradient whose last columns are padding (n_valid < N: the w2 gradient, n_valid = F), staged
    # (n_valid on 16 bytes) and direct: the addend out of place and in place, and atomic split-K onto the contents
    for nv in ([N - 8, N - 3] if N > 8 else []):
        Xv = X[:, :nv].contiguous()
        for form in ("separate", "in_place", "atomic"):
            buf = _poisoned(M, nv, r8(N) + 8, F32)
            add = buf if form == "in_place" else _poisoned(M, nv, r8(N) + 8, F32, fill=0.0)
            add[:M, :nv] = Xv

            def run(mc=0):
                buf[:M, :nv] = float("nan") if form == "separate" else Xv
                if form == "atomic":
                    lib.gemm(a, b, buf, n_valid=nv, splits=3, max_ctas=mc, **kw)
                else:
                    lib.gemm(a, b, buf, n_valid=nv, addend=add, max_ctas=mc, **kw)
            run()
            torch.cuda.synchronize()
            c5, ab5, _ = G.gemm_ref(a, b, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, n_valid=nv, out0=Xv)
            what = f"{tag} n_valid={nv} {form}"
            if form == "atomic":
                _gemm_check(buf[:M, :nv], c5, ab5, K=K, splits=3, out_dtype=F32, out0=Xv, what=what)
            else:
                _gemm_check(buf[:M, :nv], c5, ab5, K=K, out_dtype=F32, addend=Xv, what=what)
                _grid_invariant(run, buf, what)
            _guards_intact(buf, M, nv, what)
    # atomic split-K onto non-zero contents: 3 splits and more splits than k-blocks
    kb = (K + 63) // 64
    for splits in (3, kb + 2):
        buf = _poisoned(M, N, r8(N) + 8, F32, fill=0.0)
        buf[:M, :N] = X
        lib.gemm(a, b, buf, splits=splits, **kw)
        torch.cuda.synchronize()
        c4, ab4, _ = G.gemm_ref(a, b, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, out0=X)
        what = f"{tag} split-K {splits} onto X"
        _gemm_check(buf[:M, :N], c4, ab4, K=K, splits=splits, out_dtype=F32, out0=X, what=what)
        _guards_intact(buf, M, N, what)


def test_gemm16_rejects_pitches_tma_cannot_take():
    """A 16-bit operand pitch that is not a multiple of 8 elements (16 bytes) is an error on the host, for A and for B."""
    lib = _lib()
    gen = torch.Generator(device=DEV).manual_seed(0)
    M, N, K = 63, 72, 64
    a_bad = _rand((K, M), BF16, gen)                     # MN-major A with pitch 63
    b_ok = _rand((N, K), BF16, gen)
    out = torch.empty(M, N, device=DEV)
    with pytest.raises(lib.OmlmError):
        lib.gemm(a_bad, b_ok, out, a_mn=True, M=M, N=N, K=K)
    a_ok = _rand((M, K), BF16, gen)
    b_bad = _rand((K, 65), BF16, gen)                    # MN-major B with pitch 65
    with pytest.raises(lib.OmlmError):
        lib.gemm(a_ok, b_bad, out, b_mn=True, M=M, N=N, K=K)


# ------------------------------------------------------------------------------------------------ remapped weight gradients
# (sign, M, row_split, row_valid, N, n_valid): the logit head (one half of Cp rows, C live), two halves, the GEGLU order
REMAPS = [(1, 192, 192, 129, 72, 72), (1, 256, 128, 100, 136, 130), (-1, 512, -1, 200, 136, 136), (-1, 768, -1, 300, 72, 66)]


def REMAP_CASES_KEYS():
    out = []
    for sign, M, rs, rv, N, nv in REMAPS:
        for bn in (128, 256):
            for dt in (BF16, F16):
                for form in ("atomic", "in_place"):
                    out.append((sign, bn, dt, form, nv < N))
    return out


@pytest.mark.parametrize("form", ["atomic", "in_place"])
@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("remap", REMAPS, ids=[f"rs{r[2]}-rv{r[3]}-N{r[4]}-nv{r[5]}" for r in REMAPS])
def test_gemm16_remapped_weight_gradient(remap, bn, dt, form):
    """gout[rows_out, n_valid] += dy^T x with a row remap: atomic split-K onto the gradient's contents, or one split with
    the gradient as its own addend (the engine's form when the cost model picks no split)."""
    lib = _lib()
    sign, M, rs, rv, N, nv = remap
    K = 1000
    gen = torch.Generator(device=DEV).manual_seed(M + rv + bn)
    dy, x = _operand(M, K, True, dt, gen, False), _operand(N, K, True, dt, gen, False)
    rows = len(G.remap_sources(M, rs, rv))
    X = torch.randn(rows, nv, device=DEV, generator=gen)
    ldo = r8(nv) + 4
    buf = _poisoned(rows, nv, ldo, F32, extra_rows=3, fill=0.0)
    buf[:rows, :nv] = X
    kw = dict(a_mn=True, b_mn=True, M=M, N=N, K=K, row_split=rs, row_valid=rv, n_valid=nv if nv < N else 0, block_n=bn)
    if form == "atomic":
        lib.gemm(dy, x, buf, splits=4, **kw)
    else:
        lib.gemm(dy, x, buf, addend=buf, **kw)
    torch.cuda.synchronize()
    c64, ab, written = G.gemm_ref(dy, x, a_mn=True, b_mn=True, M=M, N=N, K=K, row_split=rs, row_valid=rv, n_valid=nv, out0=X)
    assert bool(written.all())
    what = f"remap {remap} bn={bn} {dt} {form}"
    if form == "atomic":
        _gemm_check(buf[:rows, :nv], c64, ab, K=K, splits=4, out_dtype=F32, out0=X, what=what, family="remap")
    else:
        _gemm_check(buf[:rows, :nv], c64, ab, K=K, out_dtype=F32, addend=X, what=what, family="remap")
        def run(mc):
            buf[:rows, :nv] = X
            lib.gemm(dy, x, buf, addend=buf, max_ctas=mc, **kw)
        _grid_invariant(run, buf, what)
    _guards_intact(buf, rows, nv, what)


# ------------------------------------------------------------------------------------------------ gemm_splitk_det
DET_CASES = [  # (M, N, K, splits, row_split, row_valid, n_valid)
    (136, 72, 64, 4, 0, 0, 0),          # one k-block: the single-split fallback (in-place addend)
    (200, 136, 1000, 5, 0, 0, 130),     # n_valid % 4 != 0
    (192, 72, 2000, 6, 192, 129, 0),    # logit head remap
    (512, 136, 1000, 3, -1, 200, 0),    # GEGLU remap
    (256, 264, 3000, 7, 128, 100, 262),
]


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("c", DET_CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}-s{c[3]}-rs{c[4]}-nv{c[6]}" for c in DET_CASES])
def test_gemm_splitk_det_per_element_and_repeatable(c, bn):
    lib = _lib()
    M, N, K, splits, rs, rv, nv0 = c
    nv = nv0 or N
    gen = torch.Generator(device=DEV).manual_seed(M + N + K + bn)
    dy, x = _operand(M, K, True, BF16, gen, False), _operand(N, K, True, BF16, gen, False)
    rows = len(G.remap_sources(M, rs, rv))
    X = torch.randn(rows, nv, device=DEV, generator=gen)
    part = torch.empty(max(lib.gemm_splitk_det_workspace(M, N, K, splits, rs, rv, nv0) // 4, 1), device=DEV)
    ldo = nv + 1
    results = []
    for mc in (0, 0, 1, 2, 7):
        buf = _poisoned(rows, nv, ldo, F32, extra_rows=3, fill=0.0)
        buf[:rows, :nv] = X
        lib.gemm_splitk_det(dy, x, buf, part, a_mn=True, b_mn=True, M=M, N=N, K=K, splits=splits, row_split=rs, row_valid=rv,
                            n_valid=nv0, block_n=bn, max_ctas=mc)
        torch.cuda.synchronize()
        results.append(buf)
    c64, ab, _ = G.gemm_ref(dy, x, a_mn=True, b_mn=True, M=M, N=N, K=K, row_split=rs, row_valid=rv, n_valid=nv, out0=X)
    what = f"splitk_det {c} bn={bn}"
    _gemm_check(results[0][:rows, :nv], c64, ab, K=K, splits=splits, out_dtype=F32, out0=X, what=what, family="splitk_det")
    _guards_intact(results[0], rows, nv, what)
    assert all(torch.equal(results[0], r) for r in results[1:]), f"{what}: repeated calls / max_ctas differ"


# ------------------------------------------------------------------------------------------------ gemm16_rowstat's output
@pytest.mark.parametrize("M,N,K", [(1000, 512, 520), (4100, 768, 256), (2048, 2816, 1024), (300, 256, 72)])
def test_gemm16_rowstat_output_per_element(M, N, K):
    lib = _lib()
    gen = torch.Generator(device=DEV).manual_seed(M + N + K)
    a = _rand((M, K), BF16, gen)
    b = _rand((K, N), BF16, gen)
    hn = _rand((M, N), BF16, gen)
    gamma = torch.randn(N, device=DEV, generator=gen)
    part = torch.full((M * (N // 128) * 2,), float("nan"), device=DEV)
    buf = _poisoned(M, N, N, BF16)
    out = buf[:M]
    lib.gemm_rowstat(a, b, out, hn, gamma, part, b_mn=True, M=M, N=N, K=K)
    torch.cuda.synchronize()
    c64, ab, _ = G.gemm_ref(a, b, b_mn=True, M=M, N=N, K=K)
    _gemm_check(out, c64, ab, K=K, out_dtype=BF16, what=f"rowstat {M}x{N}x{K}", family="rowstat")
    _guards_intact(buf, M, N, "rowstat")
    ref = out.clone()
    for mc in (1, 7):
        out.fill_(float("nan"))
        lib.gemm_rowstat(a, b, out, hn, gamma, part, b_mn=True, M=M, N=N, K=K, max_ctas=mc)
        torch.cuda.synchronize()
        assert torch.equal(out, ref), f"rowstat max_ctas={mc}"


# ------------------------------------------------------------------------------------------------ decode GEMMs
DEC_SHAPES = [(n, k) for n in (72, 200, 1088) for k in (72, 256, 520, 1032, 1152)]
DEC_B = [("skinny", B, False) for B in range(1, 17)] + \
        [("decode", B, inv) for B in (1, 16, 17, 64, 65, 128, 129, 256) for inv in (False, True)]
DEC_FORMS = [(od, add) for od in (F32, BF16, F16) for add in (False, True)]     # output type x addend


def decode_cases(B):
    """(N, K, wdt, prologue, out dtype, addend, ld_extra) of one test_decode_gemm_per_element item: every shape, weight
    format and prologue that applies to K (prologue 3 needs K % 128 == 0), with (out, addend) cycling per (prologue,
    format) so that each prologue meets all six output / addend forms in both formats (prologue 3 has exactly six
    shapes).  The offset moves with B, so different items pair forms with different shapes."""
    count = {}
    out = []
    for N, K in DEC_SHAPES:
        for wdt in (F16, BF16):
            for prologue in ((0, 1, 2, 3) if K % 128 == 0 else (0, 1, 2)):
                c = count.get((prologue, wdt), 0)
                count[(prologue, wdt)] = c + 1
                od, add = DEC_FORMS[(c + B) % len(DEC_FORMS)]
                ld_extra = (0, 8, 2)[(c + B) % 3] if prologue == 0 else ((c + B) % 2) * 4
                out.append((N, K, wdt, prologue, od, add, ld_extra))
    return out


def decode_key(entry, prologue, wdt, od, add, invariant):
    return (entry, prologue, str(wdt), str(od), bool(add), bool(invariant))


def explicit_decode_keys():
    """Keys of every decode GEMM form test_decode_gemm_per_element issues."""
    return {decode_key("skinny_gemm" if e == "skinny" else "decode_gemm", p, w, o, a, inv)
            for e, B, inv in DEC_B for (_, _, w, p, o, a, _) in decode_cases(B)}


def _decode_inputs(B, N, K, wdt, gen, big=False):
    W = (torch.randn(N, K, device=DEV, generator=gen) / K ** 0.5 * (300.0 if big else 1.0)).to(wdt)
    x = torch.randn(B, K, device=DEV, generator=gen) * 2 + 0.3
    x[::2] = 0.5 + torch.randn(x[::2].shape, device=DEV, generator=gen) * 1e-2     # var ~ 1e-4 rows: eps matters
    if big:
        x = x * 300.0
    gamma = 1 + 0.1 * torch.randn(K, device=DEV, generator=gen)
    res = torch.randn(B, N, device=DEV, generator=gen)
    return W, x, gamma, res


def _prologue_inputs(prologue, B, K, wdt, x, gamma, gen, ld_extra=0, n_real=0):
    """(A, kwargs) of a prologue.  ld_extra > 0: A is the first K columns of [B, K + ld_extra].  Prologue 3: n_real real
    channels of K (0: K - 86), the rest zero in h and gamma."""
    kw = {}
    if prologue in (0, 3):
        src = x
        if prologue == 3:
            F = n_real or K - 86
            src = torch.zeros(B, K, device=DEV)
            src[:, :F] = torch.randn(B, F, device=DEV, generator=gen) * 3 + 1
            g3 = gamma.clone()
            g3[F:] = 0
            kw = dict(gamma=g3, rowsum=torch.stack([src.view(B, -1, 128).sum(-1), (src ** 2).view(B, -1, 128).sum(-1)], -1).contiguous(), n_real=F)
        buf = torch.zeros(B, K + ld_extra, device=DEV, dtype=wdt)
        buf[:, :K] = src.to(wdt)
        return buf[:, :K], kw
    if prologue == 2:
        kw = dict(gamma=gamma)
    buf = torch.zeros(B, K + ld_extra, device=DEV)
    buf[:, :K] = x
    return buf[:, :K], kw


def _check_decode(entry, A, W, out, prologue, kw, *, addend, ws=None, invariant=False, what):
    B, (N, K) = A.shape[0], W.shape
    wdt = W.dtype
    y, e = G.decode_operand(A, prologue, wdt, gamma_=kw.get("gamma"), rowsum=kw.get("rowsum"), n_real=kw.get("n_real", 0))
    a_ref = G.round16(y, wdt)
    eop = G.operand_bound(y, e, wdt) if prologue else torch.zeros_like(y)     # prologue 0: the operand is A itself
    kb = (K + 63) // 64
    if entry == "skinny":
        gacc, splits = G.gamma_skinny(K), 1
    else:
        gacc, splits = G.gamma(18 * 4 * kb), kb        # any K split the plan picks: at most kb splits of at most kb blocks
    in_place = entry == "decode" and prologue == 0 and A.data_ptr() % 16 == 0 and A.stride(0) % 8 == 0
    if entry == "decode" and not in_place:
        a16 = ws.a16[:B * K].view(wdt).view(B, K).double()
        _note(f"decode a16 prologue {prologue}",
              G.check(a16, y if prologue else a_ref, G.operand_bound(y, e, wdt) if prologue else torch.zeros_like(y), f"{what}: a16 operand"))
        c64, ab = G.decode_ref(a16, W, addend=addend)
        extra = 0.0
    else:
        c64, ab = G.decode_ref(y, W, addend=addend)
        extra = eop @ W.double().abs().t()                 # the operand's rounding and fp32 error, carried through the products
    c64 = G.clamp_out(c64, out.dtype)
    bnd = G.decode_bound(c64, ab, K=K, out_dtype=out.dtype, gamma_acc=gacc, splits=splits, addend=addend) + extra * G.SECOND_ORDER
    return _note(f"{entry}_gemm", G.check(out, c64, bnd, what))


@pytest.mark.parametrize("entry,B,invariant", DEC_B, ids=[f"{e}-B{b}{'-inv' if i else ''}" for e, b, i in DEC_B])
def test_decode_gemm_per_element(entry, B, invariant):
    lib = _lib()
    gen = torch.Generator(device=DEV).manual_seed(B * 7919 + invariant)
    ws = lib.DecodeWorkspace(DEV, B, DEC_SHAPES, invariant=invariant) if entry == "decode" else None
    for N, K, wdt, prologue, od, has_add, ld_extra in decode_cases(B):
        W, x, gamma, res = _decode_inputs(B, N, K, wdt, gen)
        addend = res if has_add else None
        A, kw = _prologue_inputs(prologue, B, K, wdt, x, gamma, gen, ld_extra)
        out = torch.full((B, N + 3), float("nan"), device=DEV, dtype=od)
        o = out[:, :N]
        if entry == "skinny":
            lib.skinny_gemm(A, W, o, prologue=prologue, addend=addend, **kw)
        else:
            lib.decode_gemm(A, W, o, prologue=prologue, addend=addend, ws=ws, invariant=invariant, **kw)
        torch.cuda.synchronize()
        what = f"{entry} B={B} inv={invariant} N={N} K={K} {wdt} prologue={prologue} out={od} lda={A.stride(0)} addend={has_add}"
        _check_decode(entry, A, W, o, prologue, kw, addend=addend, ws=ws, invariant=invariant, what=what)
        assert bool(torch.isnan(out[:, N:]).all()), f"{what}: columns past N written"


@pytest.mark.parametrize("entry", ["skinny", "decode"])
def test_decode_gemm_fp16_clamp(entry):
    """Outputs past the fp16 range store +-65504 (the kernels clamp before the conversion)."""
    lib = _lib()
    gen = torch.Generator(device=DEV).manual_seed(5)
    B, N, K = (8 if entry == "skinny" else 40), 200, 520
    W, x, gamma, res = _decode_inputs(B, N, K, F16, gen, big=True)
    ws = lib.DecodeWorkspace(DEV, B, [(N, K)]) if entry == "decode" else None
    o = torch.full((B, N), float("nan"), device=DEV, dtype=F16)
    if entry == "skinny":
        lib.skinny_gemm(x, W, o, prologue=1)
    else:
        lib.decode_gemm(x, W, o, prologue=1, ws=ws)
    torch.cuda.synchronize()
    assert int((o.abs() == 65504).sum()) > 10, "the case must reach the clamp"
    _check_decode(entry, x, W, o, 1, {}, addend=None, ws=ws, what=f"{entry} fp16 clamp")


@pytest.mark.parametrize("prologue", [0, 3])
@pytest.mark.parametrize("entry", ["skinny", "decode"])
def test_decode_gemm_rejects_unaligned_16bit_rows(entry, prologue):
    """Prologues 0 and 3 read A in 32-bit words: an odd pitch or an odd element offset is refused on the host."""
    lib = _lib()
    B, N, K = 4, 72, 256
    W = torch.zeros(N, K, device=DEV, dtype=BF16)
    out = torch.empty(B, N, device=DEV)
    kw = {}
    if prologue == 3:
        kw = dict(gamma=torch.ones(K, device=DEV), rowsum=torch.ones(B, K // 128, 2, device=DEV), n_real=K)
    odd_pitch = torch.zeros(B, K + 1, device=DEV, dtype=BF16)[:, :K]
    odd_offset = torch.zeros(B * K + 1, device=DEV, dtype=BF16)[1:].view(B, K)
    fn = lib.skinny_gemm if entry == "skinny" else lib.decode_gemm
    for A in (odd_pitch, odd_offset):
        with pytest.raises(lib.OmlmError, match="4-byte aligned"):
            fn(A, W, out, prologue=prologue, **kw)


# ------------------------------------------------------------------------------------------------ the engine's call forms
class _Recorder:
    """Wraps the GEMM entry points of lib (the engine looks them up as module attributes at call time) and records each
    call's form: dtypes, shapes, pitches, pointer alignment and flags -- everything but the values."""

    def __init__(self, lib):
        self.lib, self.forms, self.phase, self.seen = lib, {}, None, set()
        self.orig = {n: getattr(lib, n) for n in ("gemm", "gemm_splitk_det", "gemm_rowstat", "skinny_gemm", "decode_gemm")}

    def _add(self, form):
        self.forms.setdefault(form[0], set()).add(form[1])
        self.seen.add((self.phase, form[0]))

    def __enter__(self):
        lib, o = self.lib, self.orig

        def gemm(a, b, out, *, a_mn=False, b_mn=False, M=None, N=None, K=None, addend=None, alpha=1.0, splits=1, row_split=0,
                 row_valid=0, n_valid=0, block_n=128, max_ctas=0):
            M_ = M if M is not None else (a.shape[1] if a_mn else a.shape[0])
            K_ = K if K is not None else (a.shape[0] if a_mn else a.shape[1])
            N_ = N if N is not None else (b.shape[1] if b_mn else b.shape[0])
            add = None if addend is None else ("in_place" if addend.data_ptr() == out.data_ptr() else "separate")
            self._add(("gemm", (a.dtype, a_mn, b_mn, M_, N_, K_, a.stride(0), b.stride(0), a.data_ptr() % 16, b.data_ptr() % 16,
                                out.dtype, out.stride(0), out.data_ptr() % 16, add, None if addend is None else addend.stride(0),
                                None if addend is None else addend.data_ptr() % 16, float(alpha), splits, row_split, row_valid,
                                n_valid, block_n, max_ctas)))
            return o["gemm"](a, b, out, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, addend=addend, alpha=alpha, splits=splits,
                             row_split=row_split, row_valid=row_valid, n_valid=n_valid, block_n=block_n, max_ctas=max_ctas)

        def gemm_splitk_det(a, b, out, part, *, a_mn=False, b_mn=False, M, N, K, splits, row_split=0, row_valid=0, n_valid=0,
                            block_n=128, max_ctas=0):
            self._add(("gemm_splitk_det", (a.dtype, a_mn, b_mn, M, N, K, a.stride(0), b.stride(0), out.stride(0), splits, row_split,
                                           row_valid, n_valid, block_n, max_ctas)))
            return o["gemm_splitk_det"](a, b, out, part, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, splits=splits, row_split=row_split,
                                        row_valid=row_valid, n_valid=n_valid, block_n=block_n, max_ctas=max_ctas)

        def gemm_rowstat(a, b, out, hn, gamma, part, *, b_mn=False, M=None, N=None, K=None, keep_bits=None, keep_scale=1.0, max_ctas=0):
            self._add(("gemm_rowstat", (a.dtype, b_mn, M, N, K, max_ctas)))
            return o["gemm_rowstat"](a, b, out, hn, gamma, part, b_mn=b_mn, M=M, N=N, K=K, keep_bits=keep_bits, keep_scale=keep_scale,
                                     max_ctas=max_ctas)

        def skinny_gemm(A, W, out, *, prologue=0, gamma=None, rowsum=None, n_real=0, addend=None):
            self._add(("skinny_gemm", (A.shape[0], W.shape[0], W.shape[1], W.dtype, prologue, out.dtype, addend is not None,
                                       A.stride(0), n_real)))
            return o["skinny_gemm"](A, W, out, prologue=prologue, gamma=gamma, rowsum=rowsum, n_real=n_real, addend=addend)

        def decode_gemm(A, W, out, *, prologue=0, gamma=None, rowsum=None, n_real=0, addend=None, ws=None, invariant=False):
            self._add(("decode_gemm", (A.shape[0], W.shape[0], W.shape[1], W.dtype, prologue, out.dtype, addend is not None,
                                       A.stride(0), n_real, invariant)))
            return o["decode_gemm"](A, W, out, prologue=prologue, gamma=gamma, rowsum=rowsum, n_real=n_real, addend=addend, ws=ws,
                                    invariant=invariant)

        for n, f in (("gemm", gemm), ("gemm_splitk_det", gemm_splitk_det), ("gemm_rowstat", gemm_rowstat), ("skinny_gemm", skinny_gemm),
                     ("decode_gemm", decode_gemm)):
            setattr(lib, n, f)
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(self.lib, n, f)


def _record(act16, model, monkeypatch):
    """Forms of every phase of call_forms: training steps, eval_loss, generate at B <= 16 and B > 16, and sessions."""
    with _Recorder(_lib()) as rec:
        call_forms.run(rec, model, act16, monkeypatch)
    # the shim sees the engine only while it calls through lib's attributes: every path must have shown up
    if model in call_forms.SONGS_ONLY:
        expected = {("song session", "gemm"), ("song session", "decode_gemm"), ("score songs", "gemm")}
    elif model in call_forms.BENCH_MODELS:
        expected = {(p, "gemm") for p in call_forms.BENCH_PHASES} | {("bench step", "gemm_rowstat"),
                                                                     ("bench deterministic step", "gemm_splitk_det")}
        if model in call_forms.GENERATION_MODELS:
            expected |= {("bench generation", "gemm"), ("bench generation", "skinny_gemm")}
    else:
        expected = {(p, "gemm") for p in call_forms.SESSION_PHASES} | {(p, "decode_gemm") for p in call_forms.SESSION_PHASES}
    if model in call_forms.SCORE_MODELS:
        expected.add(("score", "gemm"))
    if model in call_forms.MODELS and model not in call_forms.SESSIONS_ONLY:
        expected |= {("default step", "gemm"), ("default step", "gemm_rowstat"), ("deterministic step", "gemm"),
                     ("deterministic step", "gemm_splitk_det"), ("generate B=3", "gemm"), ("generate B=3", "skinny_gemm"),
                     ("generate B=20", "decode_gemm"), ("generate sampling", "skinny_gemm"), ("generate sampling", "decode_gemm")}
    assert expected <= rec.seen, f"entry points the engine did not call through lib: {sorted(expected - rec.seen)}"
    return rec.forms


def _replay_gemm(f, gen):
    """One recorded omlm_gemm16 form at its shape, pitches and pointer alignment, with fresh operands; returns its key."""
    lib = _lib()
    (dt, a_mn, b_mn, M, N, K, lda, ldb, pa, pb, od, ldo, po, add, ldadd, padd, alpha, splits, rs, rv, nv0, bn, mc) = f
    nv = nv0 if 0 < nv0 < N else N

    def mk(rows, cols_ld, dtype, mis):
        off = mis // (2 if dtype != F32 else 4)
        flat = (torch.randn(rows * cols_ld + off + 8, device=DEV, generator=gen)).to(dtype)
        return flat[off:off + rows * cols_ld].view(rows, cols_ld)

    a = mk(K if a_mn else M, lda, dt, pa)
    b = mk(K if b_mn else N, ldb, dt, pb)
    rows = len(G.remap_sources(M, rs, rv))
    out = mk(rows + 2, ldo, od, po)
    out.fill_(SENT)
    X = torch.randn(rows, nv, device=DEV, generator=gen)
    atomic = splits > 1
    addend = None
    if add == "in_place" or atomic:
        out[:rows, :nv] = X.to(od)
    else:
        out[:rows, :nv] = float("nan")
    if add == "in_place":
        addend = out
    elif add == "separate":
        addend = mk(rows, ldadd, F32, padd)
        addend[:, :nv] = X
    lib.gemm(a, b, out, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, addend=addend, alpha=alpha, splits=splits, row_split=rs,
             row_valid=rv, n_valid=nv0, block_n=bn, max_ctas=mc)
    torch.cuda.synchronize()
    X = X.to(od).float()
    c64, ab, written = G.gemm_ref(a, b, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, alpha=alpha, row_split=rs, row_valid=rv, n_valid=nv,
                                  addend=X if add is not None else None, out0=X if atomic else None)
    what = f"engine form {f}"
    assert bool(written.all()), f"{what}: output rows without a source row"
    _gemm_check(out[:rows, :nv], c64, ab, K=K, splits=splits, out_dtype=od, addend=X if add else None,
                out0=X if atomic else None, what=what, family="engine forms")
    _guards_intact(out, rows, nv, what)
    staged = staged_path(out_dtype=od, ldo=ldo, out_ptr=po, addend_ld=ldadd if add else None, addend_ptr=padd, atomic=atomic,
                         row_split=rs, n_valid=nv)
    return gemm_key(dt=dt, a_mn=a_mn, b_mn=b_mn, block_n=bn, out_dtype=od, addend=add or "none", atomic=atomic, row_split=rs,
                    nv_short=nv < N, staged=staged)


def _replay_decode(entry, f, gen):
    lib = _lib()
    if entry == "skinny_gemm":
        B, N, K, wdt, prologue, od, has_add, lda, n_real = f
        inv = False
    else:
        B, N, K, wdt, prologue, od, has_add, lda, n_real, inv = f
    W, x, gamma, res = _decode_inputs(B, N, K, wdt, gen)
    A, kw = _prologue_inputs(prologue, B, K, wdt, x, gamma, gen, lda - K, n_real=n_real)
    ws = lib.DecodeWorkspace(DEV, B, [(N, K)], invariant=inv) if entry == "decode_gemm" else None
    o = torch.full((B, N), float("nan"), device=DEV, dtype=od)
    addend = res if has_add else None
    if entry == "skinny_gemm":
        lib.skinny_gemm(A, W, o, prologue=prologue, addend=addend, **kw)
    else:
        lib.decode_gemm(A, W, o, prologue=prologue, addend=addend, ws=ws, invariant=inv, **kw)
    torch.cuda.synchronize()
    _check_decode("skinny" if entry == "skinny_gemm" else "decode", A, W, o, prologue, kw, addend=addend, ws=ws, what=f"engine form {entry} {f}")
    return decode_key(entry, prologue, wdt, od, has_add, inv)


def _replay_splitk_det(f, gen):
    lib = _lib()
    dt, a_mn, b_mn, M, N, K, lda, ldb, ldo, splits, rs, rv, nv0, bn, mc = f
    assert a_mn and b_mn, f
    nv = nv0 if 0 < nv0 < N else N
    dy = _rand((K, lda), dt, gen)
    x = _rand((K, ldb), dt, gen)
    rows = len(G.remap_sources(M, rs, rv))
    X = torch.randn(rows, nv, device=DEV, generator=gen)
    part = torch.empty(max(lib.gemm_splitk_det_workspace(M, N, K, splits, rs, rv, nv0) // 4, 1), device=DEV)
    buf = _poisoned(rows, nv, ldo, F32, fill=0.0)
    buf[:rows, :nv] = X
    lib.gemm_splitk_det(dy, x, buf, part, a_mn=True, b_mn=True, M=M, N=N, K=K, splits=splits, row_split=rs, row_valid=rv,
                        n_valid=nv0, block_n=bn, max_ctas=mc)
    torch.cuda.synchronize()
    c64, ab, written = G.gemm_ref(dy, x, a_mn=True, b_mn=True, M=M, N=N, K=K, row_split=rs, row_valid=rv, n_valid=nv, out0=X)
    assert bool(written.all())
    what = f"engine form gemm_splitk_det {f}"
    _gemm_check(buf[:rows, :nv], c64, ab, K=K, splits=splits, out_dtype=F32, out0=X, what=what, family="engine forms")
    _guards_intact(buf, rows, nv, what)
    return ("gemm_splitk_det", str(dt), a_mn, b_mn, bn, (rs > 0) - (rs < 0), nv < N)


@pytest.mark.parametrize("model", call_forms.MODEL_KEYS)
@pytest.mark.parametrize("act16", ["fp16", "bf16"])
def test_engine_call_forms_replayed_and_covered(act16, model, monkeypatch):
    forms = _record(act16, model, monkeypatch)
    gen = torch.Generator(device=DEV).manual_seed(17)
    covered, keys = explicit_gemm_keys(), set()
    for f in sorted(forms.get("gemm", ()), key=repr):
        keys.add(_replay_gemm(f, gen))
    for f in sorted(forms.get("gemm_splitk_det", ()), key=repr):
        keys.add(_replay_splitk_det(f, gen))
    covered |= {("gemm_splitk_det", str(BF16), True, True, bn, (c[4] > 0) - (c[4] < 0), 0 < c[6] < c[1])
                for c in DET_CASES for bn in (128, 256)}
    for f in forms.get("gemm_rowstat", ()):
        keys.add(("gemm_rowstat", str(f[0])))
    covered.add(("gemm_rowstat", str(BF16)))          # test_gemm16_rowstat_output_per_element
    for entry in ("skinny_gemm", "decode_gemm"):
        for f in sorted(forms.get(entry, ()), key=repr):
            keys.add(_replay_decode(entry, f, gen))
    covered |= explicit_decode_keys()
    print(f"act16={act16} {model}: {len(keys)} keys issued by the engine")
    for k in sorted(keys, key=repr):
        print("   ", k)
    missing = sorted((k for k in keys if k not in covered), key=repr)
    assert not missing, f"engine call forms without an explicit case: {missing}"

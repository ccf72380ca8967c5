"""The relative-position-bias path against float64 (tests/relpos_reference.py): its kernels, the engine's table and the
MLP's parameter gradients, at the precision the path claims.

The two hidden Hr x Hr layers of the continuous bias MLP run on the wgmma GEMM with bf16x3-split operands (a x ~ a_hi
w_hi + a_hi w_lo + a_lo w_hi, fp32 accumulation); forward and backward must be fp32-class, because the table reaches
|b| ~ 100 and dominates the logits.  Every tensor gets two checks:
  (i)  componentwise, |got - ref| <= 2^-12 S, with S the componentwise scale of relpos_reference.magnitude.  Derived, not
       measured: x = hi + lo + e with |e| <= 2^-16 |x|, so one bf16x3 product errs by about 3 2^-16 |a||w|.  It catches
       local garbage (a wrong tile, an unwritten tail, a misplaced third), not a dropped cross term, whose error has a
       random sign and grows like sqrt(K) while S grows like K.
  (ii) the relative L2 error of each block against the block's own norm (as in test_attention_reference_gpu.py): 128
       distances x one head of the table, 128 x 128 tiles of the matrices, whole bias vectors.  BOUNDS are about twice
       the worst value measured over every case of this file on an H100 80GB HBM3 (700 W power limit): table 1.30e-4
       (d = 1024, N = 2048), hidden-layer outputs z_1, z_2 6.0e-6, the bf16x3 GEMMs alone 5.4e-6, weight gradients
       1.5e-5 (net.3) to 2.0e-4 (net.1 at d = 72, N = 1000), bias gradients of the hidden layers up to 8.3e-4 (zero-sum
       dT: the colsum of dz cancels).  The mutation cases (dropping a_hi w_lo from the forward, a_lo from a weight
       gradient) must raise the error MUTATION_MARGIN times above the correct one (see d. below), so a lost cross term,
       swapped layout or plain-bf16 operand cannot pass.
The bias MLP's thin layers (1 -> Hr in, Hr -> heads out, and their weight gradients) run on omlm_sgemm_small and, in
deterministic mode, omlm_sgemm_small_det; the engine-level cases check them through the table and the gradients.
The t5 and 'none' tables and their backward are exact, and the d = 72 model (Hr = 36, thirds padded to 40 columns) runs
end to end against the CPU oracle."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
sys.path.insert(0, os.path.dirname(__file__))
import relpos_reference as RP  # noqa: E402

SAFE = 2.0 ** -12               # bound (i), in units of S
U32 = 2.0 ** -24
FLOOR = 0.1                     # block norms below FLOOR x the RMS block norm of the reference count as FLOOR x RMS
MUTATION_MARGIN = 16
# bound (ii) per tensor: worst block rel-L2 (see the module docstring for where they come from)
BOUNDS = {
    "gemm_fwd": 1.1e-5, "gemm_dgrad": 1e-5, "gemm_wgrad": 1.1e-5,
    "z0": 1e-7, "a0": 1e-7, "z1": 1.1e-5, "a1": 1.2e-7, "z2": 1.2e-5, "a2": 1e-7, "table": 2.7e-4,
    "net.0.0.weight": 3.2e-4, "net.0.0.bias": 1.1e-3, "net.1.0.weight": 4.1e-4, "net.1.0.bias": 1.3e-3,
    "net.2.0.weight": 3.7e-4, "net.2.0.bias": 1.7e-3, "net.3.weight": 3.1e-5, "net.3.bias": 2e-7,
    "net.3.bias zero-sum": 1.4e-8,    # absolute: ||got - ref|| / ||sum_n |dT|||
}


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as _lib
    _lib.device_check()
    return _lib


def rup8(n):
    return (n + 7) // 8 * 8


# ------------------------------------------------------------------------------------------------ error metrics
def worst_block(x, ref, br, bc):
    """2-D x, ref cut into br x bc blocks -> (worst ||x - ref|| / max(||ref||, floor) over the blocks, its block
    coordinates); floor = FLOOR x the RMS block norm of ref (1e-3 absolute where ref is all zero)."""
    x, ref = x.double(), ref.double()
    R, C = ref.shape
    nr, nc = -(-R // br), -(-C // bc)
    pad = lambda t: F.pad(t, (0, nc * bc - C, 0, nr * br - R)).reshape(nr, br, nc, bc).sum((1, 3))
    e2, r2 = pad((x - ref) ** 2), pad(ref ** 2)
    floor = FLOOR * float(r2.mean().sqrt()) or 1e-3
    err = e2.sqrt() / r2.sqrt().clamp_min(floor)
    k = int(err.argmax())
    return float(err.flatten()[k]), (k // nc, k % nc)


def blocks_of(name, t):
    if t.dim() == 1:
        return t[None], 1, t.numel()            # a bias: the whole vector
    if name == "table":
        return t, 1, 128                        # [h, N]: 128 distances of one head
    return t, 128, 128


def check(fails, name, got, ref, S, tag, extra=None, bound=None):
    """Bounds (i) and (ii) of got against ref; violations are appended to fails.  extra: an absolute allowance added to
    bound (i) (the fp32 rounding of an accumulation into a prefilled buffer).  -> the worst block error."""
    got, ref, S = got.double(), ref.double(), S.double()
    if not bool(torch.isfinite(got).all()):
        fails.append(f"{name} {tag}: non-finite values")
        return float("inf")
    allow = SAFE * S + (0.0 if extra is None else extra)
    err = (got - ref).abs()
    bad = err > allow
    ratio = float((err / allow.clamp_min(1e-300)).max())
    x, br, bc = blocks_of(name, got)
    r, _, _ = blocks_of(name, ref)
    worst, at = worst_block(x, r, br, bc)
    bound = BOUNDS[name] if bound is None else bound
    print(f"METRIC {name} {tag}: worst block {worst:.3e} at {at} (bound {bound:.1e}), componentwise {ratio:.3e} of 2^-12 S")
    if bool(bad.any()):
        idx = tuple(int(c) for c in bad.nonzero()[0])
        fails.append(f"{name} {tag}: {int(bad.sum())} entries beyond 2^-12 S, first at {idx}: got {float(got[idx]):.6e} "
                     f"ref {float(ref[idx]):.6e} S {float(S[idx]):.3e}")
    if not worst < bound:
        fails.append(f"{name} {tag}: block {at} error {worst:.3e} >= {bound:.1e}")
    return worst


# ------------------------------------------------------------------------------------------------ a. building blocks
BF_SENTINEL = -32767           # 0x8001 as int16: a negative bf16 subnormal no kernel writes here


def split_ref(x):
    hi = x.bfloat16()
    return hi, (x - hi.float()).bfloat16()


@pytest.mark.parametrize("R,C,ld", [(1, 1, 1), (5, 36, 36), (63, 36, 50), (130, 32, 32), (257, 96, 101), (70, 512, 512)])
@pytest.mark.parametrize("weight_mode", [False, True])
def test_split3_bit_exact(lib, R, C, ld, weight_mode):
    Cp = rup8(C)
    g = torch.Generator(device=DEV).manual_seed(R * 7 + C)
    src = torch.randn(R, ld, generator=g, device=DEV) * torch.exp2(torch.randint(-30, 30, (R, ld), generator=g, device=DEV).float())
    flat = src.view(-1)
    flat[::7] = 0.0
    flat[1::11] = -0.0
    flat[2::13] *= 1e-40 / flat[2::13].abs().clamp_min(1e-30)          # fp32 subnormals of either sign
    flat[3::17] = torch.sign(flat[3::17]) * 1e30
    flat[4::19] = -flat[4::19].abs()
    buf = torch.full((R * 3 * Cp + 256,), BF_SENTINEL, dtype=torch.int16, device=DEV)
    dst = buf[:R * 3 * Cp].view(torch.bfloat16).view(R, 3 * Cp)
    lib.split3_bf16(src[:, :C], dst, weight_mode=weight_mode)
    torch.cuda.synchronize()
    hi, lo = split_ref(src[:, :C])
    pad = torch.zeros(R, Cp - C, dtype=torch.bfloat16, device=DEV)
    thirds = [hi, lo, hi] if weight_mode else [hi, hi, lo]
    want = torch.cat([torch.cat([t, pad], 1) for t in thirds], 1)
    assert torch.equal(dst.view(torch.int16), want.view(torch.int16))
    assert bool((buf[R * 3 * Cp:] == BF_SENTINEL).all()), "split3 wrote past [R, 3 Cpad]"
    # hi + lo recovers x to 2^-16 relative (to the bf16 subnormal spacing 2^-133 at the bottom of the range)
    rec = hi.double() + lo.double()
    x = src[:, :C].double()
    assert bool(((rec - x).abs() <= 2.0 ** -16 * x.abs() + 2.0 ** -133).all())


@pytest.mark.parametrize("R,C", [(1, 1), (3, 36), (129, 96), (1000, 512)])
def test_bias_silu_against_float64(lib, R, C):
    g = torch.Generator(device=DEV).manual_seed(R + C)
    z = torch.randn(R, C, generator=g, device=DEV) * 8
    k = min(240, R * C)
    z.view(-1)[:k] = torch.linspace(-120, 120, 240, device=DEV)[:k]           # expf(-z) overflows below z = -88.7
    b = torch.randn(C, generator=g, device=DEV)
    zin = z.clone()
    a = torch.full_like(z, float("nan"))
    lib.bias_silu(z, b, a)
    assert torch.equal(z, zin + b)                                     # z += bias, in place, fp32-rounded
    zr = z.double()
    ref = F.silu(zr)
    allow = 2.0 ** -20 * ref.abs() + 2.0 ** -120
    assert bool(((a.double() - ref).abs() <= allow).all()), float(((a.double() - ref).abs() / allow).max())


@pytest.mark.parametrize("n", [1, 255, 257, 36 * 1000, 512 * 2048])
@pytest.mark.parametrize("bf16_copy", [False, True])
def test_silu_bwd_against_float64(lib, n, bf16_copy):
    g = torch.Generator(device=DEV).manual_seed(n)
    z = torch.randn(n, generator=g, device=DEV) * 8
    k = min(n, 481)
    z[:k] = torch.linspace(-120, 120, 481, device=DEV)[:k]
    dA = torch.randn(n, generator=g, device=DEV)
    dZ = torch.full_like(z, float("nan"))
    d16 = torch.empty(n, dtype=torch.bfloat16, device=DEV) if bf16_copy else None
    lib.silu_bwd(dA, z, dZ, d16)
    zr = z.double()
    s = torch.sigmoid(zr)
    ref = dA.double() * (s + zr * s * (1 - s))
    # the kernel forms 1 - s in fp32: an absolute 2^-24 on it, times |z| s
    scale = dA.double().abs() * (s + zr.abs() * s * (1 - s) + zr.abs() * s / 8) + 2.0 ** -100
    assert bool(((dZ.double() - ref).abs() <= 2.0 ** -20 * scale).all())
    if bf16_copy:
        assert torch.equal(d16, dZ.bfloat16())


@pytest.mark.parametrize("M,N", [(1, 1), (2, 3), (129, 8), (2048, 16), (1000, 36), (2048, 512)])
@pytest.mark.parametrize("layout", ["dtable", "rows"])
@pytest.mark.parametrize("accumulate", [False, True])
def test_colsum_against_float64(lib, M, N, layout, accumulate):
    """The engine's two uses: sum over distances of dT [h, N] (strides (1, N)) and over rows of dz [N, Hr] (strides
    (Hr, 1))."""
    g = torch.Generator(device=DEV).manual_seed(M * 3 + N)
    if layout == "dtable":
        X = torch.randn(N, M, generator=g, device=DEV)
        s_m, s_n, ref = 1, M, X.double().sum(1)
    else:
        X = torch.randn(M, N, generator=g, device=DEV)
        s_m, s_n, ref = N, 1, X.double().sum(0)
    out0 = torch.randn(N + 8, generator=g, device=DEV)
    out = out0.clone()
    lib.colsum(X, s_m, s_n, out, M, N, accumulate=accumulate)
    if accumulate:
        ref = ref + out0[:N].double()
    scale = X.double().abs().sum(1 if layout == "dtable" else 0) + out0[:N].double().abs()
    assert bool(((out[:N].double() - ref).abs() <= 2.0 ** -18 * scale).all())
    assert torch.equal(out[N:], out0[N:])


@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 2049])
def test_arange_f32_exact(lib, n):
    out = torch.full((n + 64,), -1.0, device=DEV)
    lib.arange_f32(out[:n])
    assert torch.equal(out[:n], torch.arange(n, device=DEV, dtype=torch.float32))
    assert bool((out[n:] == -1.0).all())


def _split(lib, x, weight_mode):
    R, C = x.shape
    dst = torch.empty(R, 3 * rup8(C), dtype=torch.bfloat16, device=DEV)
    lib.split3_bf16(x, dst, weight_mode=weight_mode)
    return dst


GEMM_SHAPES = [(63, 32), (1000, 36), (2048, 96), (1000, 512), (2048, 512)]


@pytest.mark.parametrize("N,Hr", GEMM_SHAPES)
def test_bf16x3_gemm_forms_against_float64(lib, N, Hr):
    """The engine's three GEMM forms on split operands: z = A3 W3^T; da = dz W as three b_mn GEMMs on strided thirds
    with the running sum as addend; dW += dz^T a as three a_mn / b_mn GEMMs accumulated into a prefilled output."""
    T = rup8(Hr)
    g = torch.Generator(device=DEV).manual_seed(N + Hr)
    a = F.silu(torch.randn(N, Hr, generator=g, device=DEV) * 3)
    w = (torch.rand(Hr, Hr, generator=g, device=DEV) * 2 - 1) / Hr ** 0.5
    dz = torch.randn(N, Hr, generator=g, device=DEV)
    a3, w3, dz3 = _split(lib, a, False), _split(lib, w, True), _split(lib, dz, False)
    fails = []
    # forward
    z = torch.full((N, Hr), float("nan"), device=DEV)
    lib.gemm(a3, w3, z, block_n=128)
    check(fails, "gemm_fwd", z, a.double() @ w.double().t(), a.double().abs() @ w.double().abs().t(), f"N={N} Hr={Hr}")
    # data gradient
    dz_hi, dz_lo = dz3[:, :Hr], dz3[:, 2 * T:2 * T + Hr]
    w_hi, w_lo = w3[:, :Hr], w3[:, T:T + Hr]
    da = torch.full((N, Hr), float("nan"), device=DEV)
    lib.gemm(dz_hi, w_hi, da, b_mn=True, M=N, N=Hr, K=Hr, block_n=128)
    lib.gemm(dz_hi, w_lo, da, b_mn=True, M=N, N=Hr, K=Hr, addend=da, block_n=128)
    lib.gemm(dz_lo, w_hi, da, b_mn=True, M=N, N=Hr, K=Hr, addend=da, block_n=128)
    check(fails, "gemm_dgrad", da, dz.double() @ w.double(), dz.double().abs() @ w.double().abs(), f"N={N} Hr={Hr}")
    # weight gradient
    a_hi, a_lo = a3[:, :Hr], a3[:, 2 * T:2 * T + Hr]
    gw0 = torch.randn(Hr, Hr, generator=g, device=DEV) * float((dz.double().t() @ a.double()).std())
    gw = gw0.clone()
    for x, y in ((dz_hi, a_hi), (dz_hi, a_lo), (dz_lo, a_hi)):
        lib.gemm(x, y, gw, a_mn=True, b_mn=True, M=Hr, N=Hr, K=N, addend=gw, block_n=128)
    ref = gw0.double() + dz.double().t() @ a.double()
    check(fails, "gemm_wgrad", gw.double() - gw0.double(), ref - gw0.double(), dz.double().abs().t() @ a.double().abs(),
          f"N={N} Hr={Hr}", extra=4 * U32 * gw.double().abs())
    assert not fails, fails


# ------------------------------------------------------------------------------------------------ b. engine forward
def make_model(d, h, bias_type="continuous", seed=0):
    import open_musiclm_b200 as O
    torch.manual_seed(seed)
    m = O.create_semantic_transformer(dim=d, depth=1, heads=h, clap_codebook_size=16, semantic_codebook_size=16,
                                      num_clap_quantizers=2, attn_dropout=0.0, ff_dropout=0.0,
                                      relative_position_bias_type=bias_type)
    return m.cuda()


def engine_at(m, N):
    """The engine and a training workspace whose table has N distances (N = sum of (n_tok + 1) over the sequences)."""
    eng = m.engine
    ws = eng.workspace(eng.plan(1, [0, N - 2]), train=True)
    assert ws["table"].shape[1] == N
    eng.refresh_packed()
    return eng, ws


def scale_to_100(eng, N):
    """Scales net.3 so that max |table| ~ 100, the magnitude the table reaches in trained models."""
    t = RP.table(RP.params_of(eng.pview), N)
    f = 100.0 / float(t.abs().max())
    eng.pview[RP.PREFIX + "net.3.weight"].mul_(f)
    eng.pview[RP.PREFIX + "net.3.bias"].mul_(f)


def check_table(fails, eng, ws, N, tag):
    p = RP.params_of(eng.pview)
    return check(fails, "table", ws["table"][:, :N], RP.table(p, N), RP.magnitude(p, N)["table"], tag)


def check_stages(fails, eng, ws, N, tag):
    """Each layer on the kernels' exact input (the previous layer's fp32 output), so a failure names its stage."""
    p = RP.params_of(eng.pview)
    prev = RP.distances(N, DEV)
    for j in range(3):
        w, b = p[f"net.{j}.0.weight"], p[f"net.{j}.0.bias"]
        z_ref = prev @ w.t() + b
        z_got = ws["rp_z"][j][:N].double()
        check(fails, f"z{j}", z_got, z_ref, prev.abs() @ w.abs().t() + b.abs(), tag)
        check(fails, f"a{j}", ws["rp_a"][j][:N], F.silu(z_got), RP.SILU_SLOPE * z_got.abs(), tag)
        prev = ws["rp_a"][j][:N].double()


FWD_CASES = [(64, 8, 2, False), (64, 8, 63, False), (64, 1, 64, True), (64, 3, 65, False), (72, 3, 2, False),
             (72, 3, 129, False), (72, 8, 1000, True), (72, 16, 2048, False), (192, 16, 129, True), (192, 3, 2048, False),
             (1024, 8, 65, False), (1024, 8, 1000, True), (1024, 16, 2048, False), (1024, 1, 2048, True)]


@pytest.mark.parametrize("d,h,N,big", FWD_CASES)
def test_engine_forward_table_against_float64(d, h, N, big):
    m = make_model(d, h)
    eng, ws = engine_at(m, N)
    if big:
        scale_to_100(eng, N)
        eng.refresh_packed()
    eng.build_bias_table(ws, N)
    tag = f"d={d} h={h} N={N}" + (" |T|~100" if big else "")
    fails = []
    check_table(fails, eng, ws, N, tag)
    check_stages(fails, eng, ws, N, tag)
    assert not fails, fails


# ------------------------------------------------------------------------------------------------ c. engine backward
def make_dT(h, N, kind, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    dT = torch.randn(h, N, generator=g, device=DEV)
    if kind == "zero_sum":          # as in training: sum_j dS_ij = 0, so every head's dT sums to zero
        dT = dT - dT.mean(1, keepdim=True)
    return dT


def run_backward(eng, ws, N, dT, det, seed):
    """Prefills arena_g with known values, runs bias_table_backward -> (arena after, prefill, the 8 gradients as
    (after - prefill) in float64, a mask of the arena elements of the 8 parameters)."""
    ws["dtable"][:, :N].copy_(dT)
    ref = RP.grads(RP.params_of(eng.pview), N, dT)
    g = torch.Generator(device=DEV).manual_seed(seed)
    prefill = torch.randn(eng.arena_g.numel(), generator=g, device=DEV)
    mask = torch.zeros_like(prefill, dtype=torch.bool)
    for k in RP.KEYS:
        o, n = eng.layout[RP.PREFIX + k], ref[k].numel()
        prefill[o:o + n] *= float(ref[k].norm()) / n ** 0.5 or 1.0          # prefill at the gradient's own scale
        mask[o:o + n] = True
    eng.arena_g.copy_(prefill)
    eng.bias_table_backward(ws, N, det)
    after = eng.arena_g.clone()
    got = {k: (eng.gview[RP.PREFIX + k].double() - prefill[eng.layout[RP.PREFIX + k]:][:ref[k].numel()].view(ref[k].shape).double())
           for k in RP.KEYS}
    return after, prefill, got, mask, ref


def check_grads(fails, eng, got, after, ref, S, zero_sum, tag):
    for k in RP.KEYS:
        acc = eng.gview[RP.PREFIX + k].double().abs()
        extra = 2 * U32 * acc                                              # rounding of the add into the prefill
        if k == "net.3.bias" and zero_sum:
            # analytically zero up to dT's own rounding: absolute, against the scale sum_n |dT|
            err = float((got[k] - ref[k]).norm() / S[k].norm())
            b = BOUNDS["net.3.bias zero-sum"]
            print(f"METRIC net.3.bias zero-sum {tag}: {err:.3e} of ||sum |dT|||  (bound {b:.1e})")
            if not err < b:
                fails.append(f"net.3.bias zero-sum {tag}: {err:.3e} >= {b:.1e}")
            if bool(((got[k] - ref[k]).abs() > SAFE * S[k] + extra).any()):
                fails.append(f"net.3.bias zero-sum {tag}: beyond 2^-12 S")
            continue
        check(fails, k, got[k], ref[k], S[k], tag, extra=extra)


BWD_CASES = [(64, 8, 129), (72, 3, 2), (72, 3, 1000), (192, 16, 65), (1024, 8, 2048)]


@pytest.mark.parametrize("d,h,N", BWD_CASES)
@pytest.mark.parametrize("kind", ["gauss", "zero_sum"])
@pytest.mark.parametrize("det", [False, True])
def test_engine_backward_gradients_against_float64(d, h, N, kind, det):
    m = make_model(d, h)
    eng, ws = engine_at(m, N)
    eng.build_bias_table(ws, N)
    dT = make_dT(h, N, kind, seed=d + N)
    after, prefill, got, mask, ref = run_backward(eng, ws, N, dT, det, seed=11)
    S = RP.magnitude(RP.params_of(eng.pview), N, dT)
    tag = f"d={d} h={h} N={N} {kind} det={det}"
    fails = []
    check_grads(fails, eng, got, after, ref, S, kind == "zero_sum", tag)
    assert torch.equal(after[~mask], prefill[~mask]), "the rel-pos backward wrote outside its 8 gradients"
    if det:
        eng.arena_g.copy_(prefill)
        eng.bias_table_backward(ws, N, det)
        assert torch.equal(eng.arena_g, after), "deterministic rel-pos backward is not bit-reproducible"
    assert not fails, fails


# ------------------------------------------------------------------------------------------------ d. mutations
# Every mutation must raise the worst block error at least MUTATION_MARGIN x above the correct error of the same case and
# break bound (ii).  For the table it also lands MUTATION_MARGIN x above the bound (measured: 39-68x).  For the weight
# gradients it cannot: their bound is set by d = 72, N = 1000 with a Gaussian dT, where cancellation over the distances
# lifts the correct error to 2.0e-4 (the error the bf16x3 forward leaves in z, through silu'), while dropping a_lo
# measured 2.5e-3 to 6.0e-3 over these cases: 6-16x the bound, 28-135x the correct error.
@pytest.mark.parametrize("d,h,N", [(64, 8, 1000), (72, 8, 1000), (1024, 16, 2048)])
def test_dropping_a_cross_term_breaks_the_table_bound(d, h, N):
    """Zeroing the lo third of the packed weights [hi | lo | hi] drops a_hi w_lo from the forward GEMMs: bound (ii) on
    the table must fail by MUTATION_MARGIN x its value."""
    m = make_model(d, h)
    eng, ws = engine_at(m, N)
    eng.build_bias_table(ws, N)
    ok = check_table([], eng, ws, N, f"d={d} h={h} N={N} correct")
    T = eng.pk_rp[0].shape[1] // 3
    eng.pk_rp[0][:, T:2 * T].zero_()
    eng.build_bias_table(ws, N)
    bad = check_table([], eng, ws, N, f"d={d} h={h} N={N} without a_hi w_lo")
    print(f"METRIC mutation table d={d} h={h} N={N}: mutated / correct {bad / ok:.1f}, "
          f"mutated / bound {bad / BOUNDS['table']:.1f}")
    eng.refresh_packed(force=True)             # version-gated: an unchanged parameter set would not repack on its own
    eng.build_bias_table(ws, N)
    again = check_table([], eng, ws, N, f"d={d} h={h} N={N} restored")
    assert ok < BOUNDS["table"] and again < BOUNDS["table"]
    assert bad >= MUTATION_MARGIN * ok, (bad, ok)
    assert bad >= MUTATION_MARGIN * BOUNDS["table"], (bad, BOUNDS["table"])


@pytest.mark.parametrize("d,h,N,kind", [(64, 8, 129, "gauss"), (72, 3, 1000, "gauss"), (1024, 8, 2048, "zero_sum")])
@pytest.mark.parametrize("j", [0, 1])
def test_dropping_a_lo_breaks_the_weight_gradient_bound(j, d, h, N, kind):
    """Zeroing the lo third of the forward split of a_j ([hi | hi | lo]) drops a_lo from dW_{j+1} = dz_{j+1}^T a_j:
    bound (ii) on net.{j+1}.0.weight must fail by MUTATION_MARGIN x its value."""
    k = f"net.{j + 1}.0.weight"
    m = make_model(d, h)
    eng, ws = engine_at(m, N)
    eng.build_bias_table(ws, N)
    dT = make_dT(h, N, kind, seed=d + N)                   # the dT of the backward case of the same shape
    S = RP.magnitude(RP.params_of(eng.pview), N, dT)
    extra = lambda: 2 * U32 * eng.gview[RP.PREFIX + k].double().abs()
    _, _, got, _, ref = run_backward(eng, ws, N, dT, False, seed=11)
    ok = check([], k, got[k], ref[k], S[k], f"d={d} h={h} N={N} {kind} correct", extra=extra())
    T = ws["rp_a3"][j].shape[1] // 3
    ws["rp_a3"][j][:, 2 * T:].zero_()
    _, _, got, _, ref = run_backward(eng, ws, N, dT, False, seed=11)
    bad = check([], k, got[k], ref[k], S[k], f"d={d} h={h} N={N} {kind} without a_lo", extra=extra())
    print(f"METRIC mutation dW{j + 1} d={d} h={h} N={N} {kind}: mutated / correct {bad / ok:.1f}, "
          f"mutated / bound {bad / BOUNDS[k]:.1f}")
    assert ok < BOUNDS[k]
    assert bad >= MUTATION_MARGIN * ok, (bad, ok)
    assert bad >= BOUNDS[k], (bad, BOUNDS[k])


# ------------------------------------------------------------------------------------------------ e. t5 and none
@pytest.mark.parametrize("h,N", [(3, 2), (8, 129), (16, 2048)])
def test_t5_table_and_backward(h, N):
    m = make_model(64, h, "t5")
    eng, ws = engine_at(m, N)
    with torch.no_grad():
        eng.pview[RP.PREFIX + "relative_attention_bias.weight"].normal_()
    eng.build_bias_table(ws, N)
    w = eng.pview[RP.PREFIX + "relative_attention_bias.weight"]
    assert torch.equal(ws["table"][:, :N], w[0][:, None].expand(h, N)), "t5 table must be bucket 0 for every distance"
    dT = make_dT(h, N, "gauss", seed=N)
    ws["dtable"][:, :N].copy_(dT)
    prefill = torch.randn(eng.arena_g.numel(), generator=torch.Generator(device=DEV).manual_seed(2), device=DEV)
    eng.arena_g.copy_(prefill)
    eng.bias_table_backward(ws, N)
    gw = eng.gview[RP.PREFIX + "relative_attention_bias.weight"]
    o = eng.layout[RP.PREFIX + "relative_attention_bias.weight"]
    p0 = prefill[o:o + gw.numel()].view(gw.shape)
    want = p0[0].double() + dT.double().sum(1)
    assert bool(((gw[0].double() - want).abs() <= 1e-6 * (dT.double().abs().sum(1) + p0[0].double().abs())).all())
    assert torch.equal(gw[1:], p0[1:]), "buckets 1..31 must not change"
    keep = torch.ones_like(prefill, dtype=torch.bool)
    keep[o:o + h] = False
    assert torch.equal(eng.arena_g[keep], prefill[keep])


@pytest.mark.parametrize("h,N", [(3, 2), (8, 1000)])
def test_none_table_is_zero_and_backward_touches_nothing(h, N):
    m = make_model(64, h, "none")
    eng, ws = engine_at(m, N)
    eng.build_bias_table(ws, N)
    assert bool((ws["table"][:, :N] == 0).all())
    ws["dtable"][:, :N].copy_(make_dT(h, N, "gauss", seed=1))
    prefill = torch.randn(eng.arena_g.numel(), generator=torch.Generator(device=DEV).manual_seed(4), device=DEV)
    eng.arena_g.copy_(prefill)
    eng.bias_table_backward(ws, N)
    assert torch.equal(eng.arena_g, prefill)


# ------------------------------------------------------------------------------------------------ f. d = 72 end to end
def test_whole_model_d72_vs_oracle():
    """A model whose rel-pos width (36) is not a multiple of 8: logits, loss and every parameter gradient against the CPU
    oracle, at the bounds of test_parity_gpu.py."""
    import open_musiclm_b200 as O
    from oracle import restatement as R
    from test_parity_gpu import _forward_vs_oracle, _grads_vs_oracle
    torch.manual_seed(0)
    m = O.create_semantic_transformer(dim=72, depth=1, heads=3, clap_codebook_size=64, semantic_codebook_size=64,
                                      num_clap_quantizers=4, attn_dropout=0.0, ff_dropout=0.1)
    g = torch.Generator().manual_seed(1234)
    toks = [torch.randint(0, 64, (2, 16), generator=g), torch.randint(0, 64, (2, 281), generator=g)]
    cfg = R.semantic_cfg(dim=72, depth=1, heads=3, codebook=64, n_clap_q=4, ce_weights=[0.0, 1.0])
    m, tr, sd = _forward_vs_oracle(m, cfg, toks, [0.0, 1.0], "d72")
    _grads_vs_oracle(m, tr, sd, cfg, toks, "d72")

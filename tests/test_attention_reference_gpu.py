"""Attention kernels against a plain float64 reference, block by block.

The training kernels (attn_fwd_tc, attn_bwd_tc in its default and fixed-order modes, and the mma.sync attn_fwd / attn_bwd
wherever they accept the shape) and the decode kernels (attn_decode, attn_decode_mqa) are compared with float64 torch
written directly from transformer.py:304-331 (SURVEY B.2), on the exact bf16 / fp32 inputs the kernels read.

A kernel bug tends to be local: one stage of a ring, one window offset, the last tile of a chunk.  One rel-L2 over a
whole tensor dilutes an error confined to one of 128 tiles by sqrt(128), so every tensor is also cut into the blocks the
kernels tile it by, and the worst block, measured against its own norm, has a bound of its own (BOUNDS).  The bounds are
about twice the worst value measured over all cases of this file on an H100 80GB HBM3; the global rel-L2 bounds are
those of test_kernels_gpu.py, except where a row's probability sits on one or two keys (PEAKED)."""
import math
import types

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
LN2 = math.log(2.0)

# (worst block error, global rel-L2) per kernel and tensor; "lse2" is an absolute bound in the log2 domain.  Worst values
# measured on an H100 80GB HBM3 (700 W) over every case of this file: out 2.4e-3 (decode 3.3e-3, decode against the
# prefill forward 4.1e-3), lse2 1.7e-5, dq 3.6e-3, dK 2.5e-3, dV 1.8e-3, dtable 3.7e-3.
_BWD = {"dq": (8e-3, 1.5e-2), "dk": (6e-3, 1.5e-2), "dv": (4e-3, 1.5e-2), "dtable": (8e-3, 1.5e-2)}
BOUNDS = {
    "fwd_tc": {"out": (5e-3, 6e-3), "lse2": 4e-5},
    "fwd_mma": {"out": (5e-3, 6e-3), "lse2": 4e-5},
    "bwd_tc": _BWD,
    "bwd_tc_det": _BWD,
    "bwd_mma": _BWD,
    "decode": {"out": (7e-3, 6e-3)},
    "decode_mqa": {"out": (7e-3, 6e-3)},
    "prefill": {"out": (1e-2, 6e-3)},      # decode output against attn_fwd_tc's row n over the same cache prefix
}
# Backward bounds where rows put nearly all their probability on one or two keys (q = k, the key-0-only prefix, N <= 2).
# There dS = P (dP - D) cancels, and D = rowsum(dO * o) is formed from the bf16 forward output o that every backward
# receives: its rounding dominates (worst measured: dq 9.2e-2, dK 4.2e-2, dtable 7.7e-2, global 2.4e-2).  The wgmma
# backward in both modes and the mma.sync backward agree on those figures to three digits, so they are the shared
# rounding point, not a kernel error.
PEAKED = {"dq": (2e-1, 5e-2), "dk": (1e-1, 5e-2), "dtable": (1.6e-1, 5e-2)}
FLOOR = 0.1         # block norms below FLOOR x the RMS block norm of the reference count as FLOOR x RMS


@pytest.fixture(scope="module")
def lib():
    from open_musiclm_b200 import lib as _lib
    _lib.load()
    return _lib


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------ float64 reference
def reference(qn, kvn, table, key_mask, B, N, h, d_o=None, scale=8.0):
    """transformer.py:304-331 in float64 on the kernels' exact inputs: sim = scale q.k + table[head, i - j], key mask,
    causal mask, softmax, P V.  -> out [B, N, h*64], lse2 [B, N*h] (log2 domain) and, given d_o, dqn [B, N, h*64],
    dkvn [B, N, 128] and dtable [h, N] from autograd.  One batch element at a time, so that the [h, N, N] intermediates
    stay at a few GB.  Rows with no visible key follow the kernels' contract (out = 0, lse2 = -inf, zero gradients)
    rather than torch's uniform fill."""
    grad = d_o is not None
    i = torch.arange(N, device=qn.device)
    delta = i[:, None] - i[None, :]
    causal = delta >= 0
    tab = table[:, :N].double().requires_grad_(grad)
    out, lse2, dq, dkv = [], [], [], []
    for b in range(B):
        with torch.set_grad_enabled(grad):
            q = qn.view(B, N, h, 64)[b].double().requires_grad_(grad)
            kv = kvn.view(B, N, 128)[b].double().requires_grad_(grad)
            vis = causal if key_mask is None else causal & key_mask.view(B, N)[b].bool()[None, :]
            has = vis.any(-1)[:, None]
            sim = scale * q.permute(1, 0, 2) @ kv[:, :64].t() + tab[:, delta.clamp_min(0)]
            sim = sim.masked_fill(~vis, float("-inf")).masked_fill(~has, 0.0)
            p = sim.softmax(-1) * has
            o = p @ kv[:, 64:]                                                  # [h, N, 64]
        lse = torch.logsumexp(sim.detach(), -1).masked_fill(~has[:, 0], float("-inf")) / LN2
        out.append(o.detach().permute(1, 0, 2).reshape(N, h * 64))
        lse2.append(lse.t().reshape(N * h))
        if grad:
            o.backward(d_o.view(B, N, h, 64)[b].double().permute(1, 0, 2))
            dq.append(q.grad.reshape(N, h * 64))
            dkv.append(kv.grad)
        del sim, p, o
    res = {"out": torch.stack(out), "lse2": torch.stack(lse2)}
    if grad:
        res.update(dq=torch.stack(dq), dkv=torch.stack(dkv), dtable=tab.grad)
    return res


# ------------------------------------------------------------------------------------------------ local error metric
def worst_block(x, ref, bs):
    """x, ref [*lead, L, inner]; a block is (*lead, bs consecutive entries of L).  -> (worst ||x - ref|| / max(||ref||,
    floor) over the blocks, its coordinates (*lead, block)); floor = FLOOR x the RMS block norm of ref.  An all-zero
    reference (a gradient that vanishes exactly) compares absolutely instead."""
    x, ref = x.double(), ref.double()
    L = ref.shape[-2]
    nb = -(-L // bs)
    e2 = F.pad(((x - ref) ** 2).sum(-1), (0, nb * bs - L)).unflatten(-1, (nb, bs)).sum(-1)
    r2 = F.pad((ref ** 2).sum(-1), (0, nb * bs - L)).unflatten(-1, (nb, bs)).sum(-1)
    floor = FLOOR * float(r2.mean().sqrt())
    if floor == 0.0:
        floor = 1e-3                     # |err| up to 1e-3 absolute per block passes where the exact value is zero
    err = e2.sqrt() / r2.sqrt().clamp_min(floor)
    k = int(err.argmax())
    return float(err.flatten()[k]), tuple(int(c) for c in torch.unravel_index(torch.tensor(k), err.shape))


# tensor -> its blocks: out / dq by (batch, head, 64 positions); dk / dv by (batch, 128-key tile); dtable by (head, 128 deltas)
def _by_head_pos(x, B, N, h):
    return x.reshape(B, N, h, 64).permute(0, 2, 1, 3), 64


LAYOUT = {
    "out": _by_head_pos,
    "dq": _by_head_pos,
    "dk": lambda x, B, N, h: (x.reshape(B, N, 128)[..., :64], 128),
    "dv": lambda x, B, N, h: (x.reshape(B, N, 128)[..., 64:], 128),
    "dtable": lambda x, B, N, h: (x.reshape(h, N, 1), 128),
}


def check(fails, kernel, name, x, ref, B, N, h, tag, peaked=False):
    """Worst block and global rel-L2 of x against ref; a failure is appended to fails (every tensor of a case is
    measured before the case fails)."""
    blk_bound, glob_bound = PEAKED[name] if peaked and name in PEAKED else BOUNDS[kernel][name]
    if not bool(torch.isfinite(x).all()):
        fails.append(f"{kernel} {name} {tag}: non-finite values")
        return
    xb, bs = LAYOUT[name](x, B, N, h)
    rb, _ = LAYOUT[name](ref, B, N, h)
    worst, at = worst_block(xb, rb, bs)
    g = rel(xb, rb) if float(rb.norm()) > 0 else float((xb.double() - rb).norm())
    print(f"METRIC {kernel} {name} {tag}: worst block {worst:.3e} at {at} (bound {blk_bound:.1e}), global {g:.3e} "
          f"(bound {glob_bound:.1e})")
    if worst >= blk_bound:
        fails.append(f"{kernel} {name} {tag}: block {at} error {worst:.3e} >= {blk_bound:.1e}")
    if g >= glob_bound:
        fails.append(f"{kernel} {name} {tag}: global rel-L2 {g:.3e} >= {glob_bound:.1e}")


def check_lse2(fails, kernel, lse, ref, tag):
    dead = torch.isinf(ref)
    if not torch.equal(torch.isneginf(lse), dead):
        fails.append(f"{kernel} {tag}: lse2 must be -inf exactly on the rows with no visible key")
        return
    err = float((lse.double() - ref)[~dead].abs().max()) if bool((~dead).any()) else 0.0
    print(f"METRIC {kernel} lse2 {tag}: max abs error {err:.3e} (bound {BOUNDS[kernel]['lse2']:.1e})")
    if not err < BOUNDS[kernel]["lse2"]:
        fails.append(f"{kernel} lse2 {tag}: max abs error {err:.3e} >= {BOUNDS[kernel]['lse2']:.1e}")


# ------------------------------------------------------------------------------------------------ training kernels
def make_inputs(B, N, h, mask, bias, qk, seed):
    """bf16 qn [B*N, h*64] / kvn [B*N, 128] (unit-norm q and k), fp32 table [h, N + 40] (table_ld > N), u8 key mask or
    None, bf16 d_o.
    bias: "rand"  -- a random per-head slope plus noise (the model's regime);
          "first" -- farther keys score higher: every row's maximum lies in key tile 0 (no rescale after the first tile);
          "diag"  -- nearer keys score higher: the maximum moves into the diagonal tile (a rescale on every tile);
          "jump"  -- +-100 in 256-delta bands: neighbouring key tiles differ by 200, i.e. 288 in the log2 domain, beyond
                     the fp32 exp2 range, so the rescale underflows to 0 in both directions;
          "zero"  -- no bias.
    qk "same": q = k for every head (each row peaks on its own key)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    M, L = B * N, N + 40
    kv = torch.randn(M, 128, device=DEV, generator=g)
    kv[:, :64] = F.normalize(kv[:, :64], dim=-1)
    if qk == "same":
        q = kv[:, None, :64].expand(M, h, 64)
    else:
        q = F.normalize(torch.randn(M, h, 64, device=DEV, generator=g), dim=-1)
    qn = q.reshape(M, h * 64).bfloat16()
    kvn = kv.bfloat16()
    d = torch.arange(L, device=DEV, dtype=torch.float32)[None]
    slope = 0.15 + 0.15 * torch.rand(h, 1, device=DEV, generator=g)
    if bias == "rand":
        table = 0.05 * torch.randn(h, 1, device=DEV, generator=g) * d + 0.3 * torch.randn(h, L, device=DEV, generator=g)
    elif bias == "first":
        table = slope * d
    elif bias == "diag":
        table = -slope * d
    elif bias == "jump":
        hh = torch.arange(h, device=DEV)[:, None]
        table = torch.where((d.long() // 256 + hh) % 2 == 0, 100.0, -100.0) + 0.3 * torch.randn(h, L, device=DEV, generator=g)
    else:
        table = torch.zeros(h, L, device=DEV)
    table = table.contiguous()
    if mask is None:
        key_mask = None
    else:
        key_mask = torch.ones(B, N, device=DEV, dtype=torch.uint8)
        if mask == "rand":              # 20 % of the keys
            key_mask = (torch.rand(B, N, device=DEV, generator=g) > 0.2).to(torch.uint8)
            key_mask[:, 0] = 1
        elif mask == "tile":            # the whole key tile 128..255
            key_mask[:, 128:256] = 0
        elif mask == "key0":            # only key 0 visible over the first three quarters
            key_mask[:, 1:3 * N // 4] = 0
        elif mask == "lead":            # the leading keys: their rows see no key at all
            key_mask[:, :min(70, N // 2)] = 0
    d_o = torch.randn(M, h * 64, device=DEV, generator=g).bfloat16()
    return qn, kvn, table, key_mask, d_o


def det_ws_floats(B, N, h, T):
    """Floats of AttnBwdDetWorkspace.ws at chunk length T: units x heads x diagonal-table width (bt_config)."""
    n_rt, n_kt = -(-N * h // 64), -(-N // 128)
    units = sum((n_rt - kt * 128 * h // 64 + T - 1) // T for kt in range(n_kt))
    return max(B * units * h * ((T * 64 + h - 1) // h + 130), 1)


def heuristic_T(lib, B, N, h):
    """The chunk length(s) whose workspace size matches the one the default heuristic sizes (for the printed record)."""
    n = lib.AttnBwdDetWorkspace(DEV, B, N, h).ws.numel()
    return [T for T in range(1, -(-N * h // 64) + 1) if det_ws_floats(B, N, h, T) == n]


def run_bwd_tc(lib, inp, out, lse, B, N, h, det, dt_init):
    """attn_bwd_tc with dqn / dkvn poisoned (they must be fully overwritten) and dtable starting at dt_init."""
    qn, kvn, table, key_mask, d_o = inp
    dq = torch.full((B * N, h * 64), float("nan"), device=DEV)
    dkv = torch.full((B * N, 128), float("nan"), device=DEV)
    dt = dt_init.clone()
    dsum = torch.empty(B * N * h, device=DEV)
    lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, key_mask, dsum, dq, dkv, dt, B, N, h, det=det)
    torch.cuda.synchronize()
    return dq, dkv, dt


def check_grads(fails, kernel, dq, dkv, dtable, ref, B, N, h, tag, peaked=False):
    check(fails, kernel, "dq", dq, ref["dq"], B, N, h, tag, peaked)
    check(fails, kernel, "dk", dkv, ref["dkv"], B, N, h, tag, peaked)
    check(fails, kernel, "dv", dkv, ref["dkv"], B, N, h, tag, peaked)
    check(fails, kernel, "dtable", dtable, ref["dtable"], B, N, h, tag, peaked)


# (B, N, h, key mask, bias, q/k): sequence edges, head counts whose row tiles start mid-position (3, 12), a grid far above
# 4 CTAs per SM, the head limits with partial tail tiles (fwd 68, bwd 58), every mask and every bias regime.
CASES = [
    (1, 1, 1, None, "rand", "rand"),
    (3, 2, 3, "rand", "rand", "rand"),
    (2, 63, 8, "rand", "first", "rand"),
    (2, 64, 12, None, "diag", "rand"),
    (1, 65, 3, "lead", "rand", "rand"),
    (2, 127, 16, "rand", "diag", "rand"),
    (1, 128, 1, "rand", "jump", "rand"),
    (2, 129, 8, "key0", "rand", "rand"),
    (1, 255, 12, None, "zero", "same"),
    (2, 257, 3, "rand", "first", "rand"),
    (1, 263, 68, "rand", "rand", "rand"),
    (1, 301, 58, "rand", "diag", "rand"),
    (2, 512, 1, "tile", "jump", "rand"),
    (2, 1000, 8, "tile", "diag", "rand"),
    (1, 1000, 16, "key0", "jump", "rand"),
    (1, 2048, 8, "rand", "rand", "rand"),
    (1, 2048, 3, "lead", "jump", "rand"),
    (24, 1024, 8, "rand", "rand", "rand"),
]


@pytest.mark.parametrize("B,N,h,mask,bias,qk", CASES,
                         ids=[f"B{c[0]}-N{c[1]}-h{c[2]}-{c[3]}-{c[4]}-{c[5]}" for c in CASES])
def test_training_attention_against_float64(lib, B, N, h, mask, bias, qk):
    """Forward (out, lse2) and backward (dqn, dK, dV, dtable) of every training kernel that accepts the shape; the wgmma
    backward in both modes with dqn / dkvn poisoned and dtable accumulated onto random values in a table wider than N."""
    inp = make_inputs(B, N, h, mask, bias, qk, seed=1000 * h + N + B)
    qn, kvn, table, key_mask, d_o = inp
    M = B * N
    bwd_ok = h <= 58
    ref = reference(qn, kvn, table, key_mask, B, N, h, d_o if bwd_ok else None)
    tag = f"B={B} N={N} h={h} mask={mask} bias={bias} qk={qk}"
    peaked = qk == "same" or mask == "key0" or N <= 2
    fails, fwd = [], {}
    for kernel, fn in (("fwd_tc", lib.attn_fwd_tc), ("fwd_mma", lib.attn_fwd)):
        if kernel == "fwd_mma" and h > 29:
            continue
        out = torch.full((M, h * 64), float("nan"), device=DEV, dtype=torch.bfloat16)
        lse = torch.full((B, N * h), float("nan"), device=DEV)
        fn(qn, kvn, table, key_mask, out, lse, B, N, h)
        torch.cuda.synchronize()
        check(fails, kernel, "out", out, ref["out"].view(M, h * 64), B, N, h, tag)
        check_lse2(fails, kernel, lse, ref["lse2"], tag)
        fwd[kernel] = (out, lse)
    if not bwd_ok:
        assert not fails, "\n".join(fails)
        return
    print(f"METRIC heuristic T {tag}: {heuristic_T(lib, B, N, h)}")
    out, lse = fwd["fwd_tc"]
    rms = float(ref["dtable"].pow(2).mean().sqrt())
    dt_init = torch.randn(table.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(N)) * max(rms, 1e-3)
    ws = lib.AttnBwdDetWorkspace(DEV, B, N, h)
    for kernel, det in (("bwd_tc", None), ("bwd_tc_det", ws)):
        dq, dkv, dt = run_bwd_tc(lib, inp, out, lse, B, N, h, det, dt_init)
        assert torch.equal(dt[:, N:], dt_init[:, N:]), f"{kernel} {tag}: dtable written beyond N"
        check_grads(fails, kernel, dq, dkv, dt[:, :N] - dt_init[:, :N], ref, B, N, h, tag, peaked)
    assert not ws.error()
    # the mma.sync backward turns rows without a visible key into NaN (exp2(-inf - -inf)); only the wgmma backward
    # implements that part of the contract, and only it trains
    if h <= 16 and bool(torch.isfinite(ref["lse2"]).all()):
        o_m, lse_m = fwd["fwd_mma"]
        dq = torch.zeros(M, h * 64, device=DEV)
        dkv = torch.zeros(M, 128, device=DEV)
        dt = torch.zeros_like(table)
        lib.attn_bwd(qn, kvn, d_o, o_m, lse_m, table, key_mask, torch.empty(M * h, device=DEV), dq, dkv, dt, B, N, h)
        torch.cuda.synchronize()
        check_grads(fails, "bwd_mma", dq, dkv, dt[:, :N], ref, B, N, h, tag, peaked)
    assert not fails, "\n".join(fails)


# The training workspace's forms: a bias table exactly N wide (table_ld = N), and the backward without the bias gradient
# (a frozen or absent relative-position bias).  Shapes of the d = 72 / h = 3 and cfg2 / h = 8 training steps and prefills.
EXACT_CASES = [
    (4, 50, 3, "rand", "rand", "rand"),
    (3, 33, 3, None, "diag", "rand"),
    (20, 40, 3, "rand", "rand", "rand"),
    (4, 1024, 8, "rand", "rand", "rand"),
    (3, 230, 8, "rand", "diag", "rand"),
    (2, 100, 16, None, "rand", "rand"),
    (2, 1024, 16, "rand", "rand", "rand"),         # bench.py's cfg4 (musiclm_large): h = 16 at N = 1024
    (2, 15, 8, "rand", "rand", "rand"),            # bench.py's generation: the semantic stage's prefill of the clap ids
]


@pytest.mark.parametrize("B,N,h,mask,bias,qk", EXACT_CASES,
                         ids=[f"B{c[0]}-N{c[1]}-h{c[2]}-{c[3]}-{c[4]}-{c[5]}" for c in EXACT_CASES])
def test_exact_table_width_and_no_bias_gradient(lib, B, N, h, mask, bias, qk):
    """attn_fwd_tc and attn_bwd_tc (both modes) on a table exactly N wide against float64, and with dtable None: dqn / dkvn
    against float64, in the fixed-order mode bit-identical to the call with a table gradient."""
    qn, kvn, table, key_mask, d_o = make_inputs(B, N, h, mask, bias, qk, seed=3000 * h + N + B)
    table = table[:, :N].contiguous()
    inp = (qn, kvn, table, key_mask, d_o)
    M = B * N
    ref = reference(qn, kvn, table, key_mask, B, N, h, d_o)
    tag = f"B={B} N={N} h={h} mask={mask} bias={bias} table_ld=N"
    fails = []
    out = torch.full((M, h * 64), float("nan"), device=DEV, dtype=torch.bfloat16)
    lse = torch.full((B, N * h), float("nan"), device=DEV)
    lib.attn_fwd_tc(qn, kvn, table, key_mask, out, lse, B, N, h)
    torch.cuda.synchronize()
    check(fails, "fwd_tc", "out", out, ref["out"].view(M, h * 64), B, N, h, tag)
    check_lse2(fails, "fwd_tc", lse, ref["lse2"], tag)
    ws = lib.AttnBwdDetWorkspace(DEV, B, N, h)
    for kernel, det in (("bwd_tc", None), ("bwd_tc_det", ws)):
        dq, dkv, dt = run_bwd_tc(lib, inp, out, lse, B, N, h, det, torch.zeros_like(table))
        check_grads(fails, kernel, dq, dkv, dt, ref, B, N, h, tag)
        dq0 = torch.full_like(dq, float("nan"))
        dkv0 = torch.full_like(dkv, float("nan"))
        lib.attn_bwd_tc(qn, kvn, d_o, out, lse, table, key_mask, torch.empty(M * h, device=DEV), dq0, dkv0, None, B, N, h, det=det)
        torch.cuda.synchronize()
        for name, x, r in (("dq", dq0, ref["dq"]), ("dk", dkv0, ref["dkv"]), ("dv", dkv0, ref["dkv"])):
            check(fails, kernel, name, x, r, B, N, h, tag + " dtable=None")
        if det is not None and not (torch.equal(dq0, dq) and torch.equal(dkv0, dkv)):
            fails.append(f"{kernel} {tag}: dqn / dkvn without dtable differ from the call with it")
    assert not ws.error()
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("B,N,h", [(2, 700, 3), (1, 1024, 8), (1, 260, 12)])
def test_backward_at_forced_chunk_lengths(lib, monkeypatch, B, N, h):
    """OMLM_ATTN_BWD_T forces the backward's chunk length T (row tiles per work unit), which decides how dK|dV are
    flushed, the width and dmin of the diagonal tables and the fixed-order turns.  At T = 1, 2, 3 and all row tiles: both
    modes against float64; the fixed-order mode bit-identical over two calls; the modes within 1e-6 of each other."""
    inp = make_inputs(B, N, h, "rand", "diag", "rand", seed=7 * N + h)
    qn, kvn, table, key_mask, d_o = inp
    ref = reference(qn, kvn, table, key_mask, B, N, h, d_o)
    out = torch.empty(B * N, h * 64, device=DEV, dtype=torch.bfloat16)
    lse = torch.empty(B, N * h, device=DEV)
    lib.attn_fwd_tc(qn, kvn, table, key_mask, out, lse, B, N, h)
    monkeypatch.delenv("OMLM_ATTN_BWD_T", raising=False)
    n_rt = -(-N * h // 64)
    print(f"METRIC heuristic T B={B} N={N} h={h}: {heuristic_T(lib, B, N, h)} of {n_rt} row tiles")
    zero = torch.zeros_like(table)
    fails = []
    for T in sorted({1, 2, 3, n_rt}):
        monkeypatch.setenv("OMLM_ATTN_BWD_T", str(T))
        ws = lib.AttnBwdDetWorkspace(DEV, B, N, h)           # sized for T: proves the override took effect
        assert ws.ws.numel() == det_ws_floats(B, N, h, T), (T, ws.ws.numel())
        tag = f"B={B} N={N} h={h} T={T}"
        dflt = run_bwd_tc(lib, inp, out, lse, B, N, h, None, zero)
        det = run_bwd_tc(lib, inp, out, lse, B, N, h, ws, zero)
        again = run_bwd_tc(lib, inp, out, lse, B, N, h, ws, zero)
        assert not ws.error()
        for name, a, b, c in zip(("dq", "dkv", "dtable"), dflt, det, again):
            assert torch.equal(b, c), f"{tag}: fixed-order {name} differs between two calls"
            assert rel(a, b) < 1e-6, f"{tag}: {name} default vs fixed-order {rel(a, b):.2e}"
        for kernel, (dq, dkv, dt) in (("bwd_tc", dflt), ("bwd_tc_det", det)):
            check_grads(fails, kernel, dq, dkv, dt[:, :N], ref, B, N, h, tag)
    assert not fails, "\n".join(fails)


def test_head_limits_are_enforced(lib):
    """The shared-memory bias windows admit 68 heads in the forward and 58 in the backward (both run in
    test_training_attention_against_float64); one more is an argument error, not a launch."""
    B, N = 1, 64
    for h, fwd_ok in ((69, False), (59, True)):
        qn = torch.zeros(B * N, h * 64, device=DEV, dtype=torch.bfloat16)
        kvn = torch.zeros(B * N, 128, device=DEV, dtype=torch.bfloat16)
        table = torch.zeros(h, N, device=DEV)
        out = torch.empty_like(qn)
        lse = torch.empty(B, N * h, device=DEV)
        if fwd_ok:
            lib.attn_fwd_tc(qn, kvn, table, None, out, lse, B, N, h)
        else:
            with pytest.raises(lib.OmlmError, match="too many heads"):
                lib.attn_fwd_tc(qn, kvn, table, None, out, lse, B, N, h)
        grads = (torch.empty(B * N * h, device=DEV), torch.empty(B * N, h * 64, device=DEV), torch.empty(B * N, 128, device=DEV),
                 torch.zeros_like(table))
        fake_ws = types.SimpleNamespace(ws=torch.zeros(1, device=DEV), iws=torch.zeros(1, device=DEV, dtype=torch.int32))
        for det in (None, fake_ws):
            with pytest.raises(lib.OmlmError, match="too many heads"):
                lib.attn_bwd_tc(qn, kvn, qn, out, lse, table, None, *grads, B, N, h, det=det)
        with pytest.raises(lib.OmlmError, match="too many heads"):
            lib.AttnBwdDetWorkspace(DEV, B, N, h)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ decode kernels
MAX_POS = 1100                   # not a multiple of the 128-key slices
DECODE_N = [0, 1, 63, 127, 128, 129, 255, 256, 1000, MAX_POS - 1]
DECODE_CASES = ([("decode", B, h, n) for (B, h), n in zip([(1, 1), (5, 3), (16, 8), (5, 16)] * 3, DECODE_N)]
                + [("decode_mqa", B, h, n) for (B, h), n in zip([(17, 1), (64, 3), (17, 8), (64, 16)] * 3, DECODE_N)]
                + [("decode_mqa", 256, 8, MAX_POS - 1)])


@pytest.mark.parametrize("kernel,B,h,n", DECODE_CASES, ids=[f"{k}-B{B}-h{h}-n{n}" for k, B, h, n in DECODE_CASES])
def test_decode_attention_against_float64(lib, kernel, B, h, n):
    """One decode step at position n against float64 over keys 0..n, with q and k rounded as both kernels document
    (bf16(l2norm(x) * scale)).  Cache rows above n hold NaN, so a read past n shows as a non-finite output.  Rows below
    n stay bit-identical; the appended row n is within one bf16 ulp of torch's rounding.  The output also matches row n
    of attn_fwd_tc over the cache prefix of length n + 1 with the same bf16 query (what generate relies on)."""
    g = torch.Generator(device=DEV).manual_seed(97 * n + 13 * h + B)
    ld = MAX_POS + 40
    k_scale = 0.5 + torch.rand(64, device=DEV, generator=g)
    q_scale = 0.5 + torch.rand(64, device=DEV, generator=g)
    k = F.normalize(torch.randn(B, MAX_POS, 64, device=DEV, generator=g), dim=-1) * k_scale
    v = torch.randn(B, MAX_POS, 64, device=DEV, generator=g)
    cache = torch.cat([k, v], -1).bfloat16()
    cache[:, n:] = float("nan")
    cache0 = cache.clone()
    q_raw = (2 * torch.randn(B, h * 64, device=DEV, generator=g)).bfloat16()
    kv_raw = (2 * torch.randn(B, 128, device=DEV, generator=g)).bfloat16()
    d = torch.arange(ld, device=DEV, dtype=torch.float32)[None]
    table = (0.5 * torch.randn(h, ld, device=DEV, generator=g) - 0.01 * torch.rand(h, 1, device=DEV, generator=g) * d).contiguous()
    pos = torch.full((1,), n, device=DEV, dtype=torch.int32)
    out = torch.full((B, h * 64), float("nan"), device=DEV, dtype=torch.bfloat16)
    if kernel == "decode":
        lib.attn_decode(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, MAX_POS, out, h)
    else:
        ws = lib.DecodeWorkspace(DEV, B, [(1, 8)], max_pos=MAX_POS, heads=h)
        lib.attn_decode_mqa(q_raw, kv_raw, q_scale, k_scale, cache, table, pos, MAX_POS, out, h, ws=ws)
    torch.cuda.synchronize()
    tag = f"B={B} h={h} n={n}"
    # the cache: rows below n untouched, row n appended, rows above n never written
    assert torch.equal(cache[:, :n], cache0[:, :n])
    assert torch.isnan(cache[:, n + 1:].float()).all()
    row = torch.cat([(F.normalize(kv_raw[:, :64].float(), dim=-1) * k_scale).bfloat16(), kv_raw[:, 64:]], -1)
    got = cache[:, n].float()
    assert ((got - row.float()).abs() <= row.float().abs() * 2.0 ** -7).all(), f"{tag}: appended row beyond one bf16 ulp"
    if kernel == "decode_mqa":
        assert int(ws.counters.abs().sum()) == 0
    # float64 reference over keys 0..n
    qn = (F.normalize(q_raw.float().view(B, h, 64), dim=-1) * q_scale).bfloat16()
    keys = torch.cat([cache0[:, :n], row[:, None]], 1).double()                 # [B, n + 1, 128]
    j = torch.arange(n + 1, device=DEV)
    sim = 8.0 * qn.double() @ keys[..., :64].transpose(1, 2) + table[:, n - j].double()[None]
    ref = sim.softmax(-1) @ keys[..., 64:]                                       # [B, h, 64]
    fails = []
    check(fails, kernel, "out", out, ref.reshape(B, h * 64), B, 1, h, tag)
    # prefill / decode: row n of the full forward over the prefix, same bf16 query
    Np = n + 1
    qfull = torch.zeros(B, Np, h * 64, device=DEV, dtype=torch.bfloat16)
    qfull[:, n] = qn.reshape(B, h * 64)
    out_f = torch.empty(B * Np, h * 64, device=DEV, dtype=torch.bfloat16)
    lse_f = torch.empty(B, Np * h, device=DEV)
    lib.attn_fwd_tc(qfull.view(B * Np, h * 64), cache[:, :Np].contiguous().view(B * Np, 128), table, None, out_f, lse_f, B, Np, h)
    torch.cuda.synchronize()
    check(fails, "prefill", "out", out, out_f.view(B, Np, h * 64)[:, n].float(), B, 1, h, tag)
    assert not fails, "\n".join(fails)

"""Float64 reference of one optimiser step on the engine's flat parameter arena, and error scales for the fp32
arithmetic of the kernels that implement it (csrc/optim.cu: sumsq_kernel, adamw_kernel).

The reference is what the reference trainer does per step (open_musiclm/trainer.py:443-449, optimizer.py:10-40):
clip_grad_norm_(max_grad_norm) over the parameters that have a gradient, then AdamW with decoupled decay on the
ndim >= 2 group (Adam when wd == 0), with the LinearLR warm-up factor and bias corrections from each parameter's own
step count.  Parameters without a gradient are skipped, as torch's optimizers skip `grad is None`.

The error scales are derived, not fitted.  Every fp32 operation of the kernel is charged u = 2^-24 of the magnitude of
its result plus ETA = 2^-150 (half the smallest subnormal: underflow), every fp32 input the reference holds in float64
(the hyper-parameters) is charged its rounding, rsqrtf its documented 2 ulp, and errors are propagated to first order
through each operation.  A kernel result outside its scale is a kernel error, not rounding.
"""
import math

import torch

U = 2.0 ** -24
ETA = 2.0 ** -150
CLIP_EPS = 1e-6              # torch.nn.utils.clip_grad_norm_: max_norm / (total_norm + 1e-6)


def gamma(k):
    return k * U / (1 - k * U)


def lr_factor(steps, warmup, start_factor=1e-7):
    """lr / base lr after `steps` scheduler steps of LinearLR(start_factor, 1.0, total_iters=warmup), by the recursion
    torch's LinearLR.get_lr applies; 1 without warm-up (the reference builds no scheduler then)."""
    if warmup <= 0:
        return 1.0
    f = start_factor
    for e in range(1, min(steps, warmup) + 1):
        f *= 1.0 + (1.0 - start_factor) / (warmup * start_factor + (e - 1) * (1.0 - start_factor))
    return f


def hyper_vector(*, t, lr, betas=(0.9, 0.99), eps=1e-8, wd=0.0, max_grad_norm=None, prescale=1.0):
    """adamw_kernel's hyper[9] (HotPathTrainer._set_hyper) in float64: lr is the scheduled learning rate."""
    b1, b2 = betas
    return [lr, b1, b2, eps, wd, 1 - b1 ** t, 1 - b2 ** t, max_grad_norm if max_grad_norm is not None else 0.0, prescale]


def live_mask(n, frozen, device=None):
    keep = torch.ones(n, dtype=torch.bool, device=device)
    for a, b in frozen:
        keep[a:b] = False
    return keep


def sumsq(g, prescale=1.0, frozen=()):
    """sum (g * prescale)^2 in float64 over the parameters with a gradient."""
    g = g.double()
    if frozen:
        g = g[live_mask(g.numel(), frozen, g.device)]
    return float((g * prescale).square().sum())


def clip_coef(norm, max_grad_norm):
    """torch.nn.utils.clip_grad_norm_'s factor; 1 without clipping (trainer max_grad_norm None)."""
    if max_grad_norm is None or max_grad_norm <= 0:
        return 1.0
    return min(1.0, max_grad_norm / (norm + CLIP_EPS))


def adamw_update(p, g, m, v, *, t, lr, wd, n_decay, betas=(0.9, 0.99), eps=1e-8, max_grad_norm=None, prescale=1.0,
                 frozen=()):
    """One update of flat arrays in float64; returns (p, m, v, norm).  g is the summed gradient (the DDP mean's
    1/world is prescale).  Decay on [0, n_decay).  t: step count, a number or one per element (torch counts per
    parameter).  frozen: arena ranges [a, b) of parameters without a gradient this step: p, m and v stay."""
    p, g, m, v = (x.double() for x in (p, g, m, v))
    b1, b2 = betas
    gs = g * prescale
    norm = math.sqrt(sumsq(gs, 1.0, frozen))
    G = gs * clip_coef(norm, max_grad_norm)
    t = torch.as_tensor(t, dtype=torch.float64, device=p.device)
    decay = torch.ones_like(p)
    decay[:n_decay] = 1.0 - lr * wd
    P = p * decay
    M = b1 * m + (1 - b1) * G
    V = b2 * v + (1 - b2) * G * G
    denom = V.sqrt() / (1 - b2 ** t).sqrt() + eps
    P = P - lr / (1 - b1 ** t) * M / denom
    live = live_mask(p.numel(), frozen, p.device)
    return torch.where(live, P, p), torch.where(live, M, m), torch.where(live, V, v), norm


def reference_optimizer(params, *, lr, wd, betas=(0.9, 0.99), eps=1e-8):
    """The optimizer the reference's get_optimizer builds (optimizer.py:10-34): Adam when wd == 0, else AdamW with
    [ndim >= 2 | the rest with weight_decay 0]."""
    params = list(params)
    if wd == 0:
        return torch.optim.Adam(params, lr=lr, betas=betas, eps=eps)
    return torch.optim.AdamW([{"params": [p for p in params if p.ndim >= 2]},
                              {"params": [p for p in params if p.ndim < 2], "weight_decay": 0}],
                             lr=lr, weight_decay=wd, betas=betas, eps=eps)


# ------------------------------------------------------------------------------------------------ kernel error scales
def sumsq_grid(n, sms):
    """(blocks, threads) of omlm_grad_sumsq / _det."""
    return min((n // 4 + 511) // 512 + 1, sms * 4), 512


def sumsq_bound(g, prescale, blocks, threads=512):
    """|kernel - exact| for grad_sumsq.  Each thread sums k = 4 ceil(n4 / (blocks threads)) squares (+1 tail element) in
    one fp32 chain, the block adds its 512 sums in a 10-level fp32 tree, the blocks' sums are added in float64.  All
    terms are >= 0, so the fp32 part errs by at most gamma(k + 11) of the sum, plus ETA per square that underflows."""
    n = g.numel()
    k = 4 * -(-(n // 4) // (blocks * threads)) + 1
    s = sumsq(g, 1.0)
    return prescale * prescale * (gamma(k + 11) * s + 2 * n * ETA + (blocks + 2) * 2.0 ** -53 * s)


def adamw_bound(p, g, m, v, *, t, lr, wd, n_decay, betas=(0.9, 0.99), eps=1e-8, max_grad_norm=None, prescale=1.0,
                sumsq_value=None, sumsq_err=0.0, frozen=()):
    """Per-element bounds (Ep, Em, Ev) on |kernel - adamw_update| for adamw_kernel on fp32 inputs p, g, m, v.
    sumsq_value / sumsq_err: the float64 sum of squares the kernel reads and its distance from the exact one."""
    p, g, m, v = (x.double() for x in (p, g, m, v))
    b1, b2 = betas
    a = torch.abs
    S = sumsq(g, prescale, frozen) if sumsq_value is None else sumsq_value
    norm = math.sqrt(S)
    # coef = prescale * min(1, max_norm / (norm + 1e-6))
    if max_grad_norm is not None and max_grad_norm > 0:
        rel_norm = (sumsq_err / (2 * S) if S > 0 else 0.0) + U
        c = max_grad_norm / (norm + CLIP_EPS)
        rel_c = U + (norm * rel_norm + CLIP_EPS * U) / (norm + CLIP_EPS) + U + U
        cmin = min(1.0, c)
        e_cmin = 0.0 if c * (1 - rel_c) >= 1 else rel_c * c
        coef = prescale * cmin
        e_coef = prescale * (e_cmin + 2 * U * cmin)
    else:
        coef, e_coef = prescale, prescale * U
    G = g * coef
    eG = a(g) * e_coef + U * a(G) + ETA
    # p * (1 - lr wd) on [0, n_decay)
    D = 1.0 - lr * wd
    eD = 3 * U * lr * wd + U * D if wd != 0 else 0.0
    dec = torch.zeros_like(p, dtype=torch.bool)
    dec[:n_decay] = True
    Pd = torch.where(dec, p * D, p)
    ePd = torch.where(dec, a(p) * eD + U * a(p * D) + ETA, torch.zeros_like(p)) if wd != 0 else torch.zeros_like(p)
    # m = b1 m + (1 - b1) g
    M = b1 * m + (1 - b1) * G
    eM = 2 * U * b1 * a(m) + U * b1 * a(G) + (1 - b1) * (eG + U * a(G)) + U * (b1 * a(m) + (1 - b1) * a(G)) + 3 * ETA
    # v = b2 v + (1 - b2) g g
    V = b2 * v + (1 - b2) * G * G
    eV = (2 * U * b2 * a(v) + U * b2 * G * G + (1 - b2) * (2 * a(G) * eG + eG * eG + 2 * U * G * G)
          + U * (b2 * a(v) + (1 - b2) * G * G) + 3 * ETA)
    # denom = sqrtf(v) rsqrtf(1 - b2^t) + eps
    R = V.sqrt()
    eR0 = torch.where(V > 0, torch.minimum(eV.sqrt(), eV / V.sqrt()), eV.sqrt())
    eR = eR0 + U * (R + eR0) + ETA
    t = torch.as_tensor(t, dtype=torch.float64, device=p.device)
    inv = 1.0 / (1 - b2 ** t).sqrt()
    rel_inv = 0.5 * U + 4 * U
    Sd = R * inv
    eS = eR * inv + Sd * rel_inv + U * Sd + ETA
    Dn = Sd + eps
    eDn = eS + eps * U + U * Dn
    # q = m / denom, p -= (lr / bc1) q
    Q = M / Dn
    eQ = eM / Dn + a(M) * eDn / (Dn * (Dn - eDn)) + U * a(Q) + ETA
    step = lr / (1 - b1 ** t)
    Up = step * Q
    eU = step * eQ + 4 * U * step * a(Q) + U * a(Up) + ETA
    eP = ePd + eU + U * (a(Pd) + a(Up)) + ETA
    live = live_mask(p.numel(), frozen, p.device)
    z = torch.zeros_like(p)
    return torch.where(live, eP, z), torch.where(live, eM, z), torch.where(live, eV, z)


def adamw_cases(n, seed, device=None):
    """fp32 (p, g, m, v) with the values where the update goes wrong: gradients at 0, subnormal, 1e-12, 1 and 1e4 of
    either sign; v = 0 with g = 0 (the denominator is exactly eps); v so small that sqrt(v) ~ eps (eps inside the square
    root would change the step by orders of magnitude); ordinary Adam states elsewhere."""
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=gen) * 0.05
    mags = torch.tensor([0.0, 1e-40, 1e-12, 1.0, 1e4])
    g = mags[torch.randint(0, len(mags), (n,), generator=gen)] * torch.randn(n, generator=gen).sign()
    g = torch.where(torch.rand(n, generator=gen) < 0.4, torch.randn(n, generator=gen), g)
    m = torch.randn(n, generator=gen) * 1e-3
    v = torch.rand(n, generator=gen) * 1e-6
    kind = torch.randint(0, 8, (n,), generator=gen)
    v = torch.where(kind == 0, torch.zeros(n), v)
    g = torch.where(kind == 0, torch.zeros(n), g)
    v = torch.where(kind == 1, torch.rand(n, generator=gen) * 1e-16, v)
    g = torch.where(kind == 1, torch.randn(n, generator=gen) * 1e-9, g)
    m = torch.where(kind == 2, torch.zeros(n), m)
    out = [x.float().contiguous() for x in (p, g, m, v)]
    return [x.to(device) for x in out] if device is not None else out

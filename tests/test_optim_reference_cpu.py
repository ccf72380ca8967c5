"""The float64 optimiser reference (tests/optim_reference.py) pinned without a GPU: against torch's AdamW / Adam,
clip_grad_norm_ and LinearLR, against the oracle's restatement, against the reference's get_optimizer where a checkout
is present; its error scales against an fp32 replica of the kernels' arithmetic; the frozen-parameter rule against the
`grad is None` sets the reference fixtures recorded."""
import glob
import importlib
import math
import os

import numpy as np
import pytest
import torch

import optim_reference as OR
from oracle import ref_harness
from oracle import restatement as R

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "tiny_*.pt")))
SHAPES = {"w1": (6, 5), "w2": (4, 3), "b": (7,), "s": (3,)}         # arena order: [ndim >= 2 | the rest]
NONE_ON = "w2"                                                      # this one has no gradient on every third step


def _layout():
    off, lay = 0, {}
    for k, s in SHAPES.items():
        lay[k] = (off, off + math.prod(s))
        off += math.prod(s)
    return lay, off, lay["b"][0]


def _grads(step, gen, scale):
    gs = {k: torch.randn(s, generator=gen, dtype=torch.float64) * scale for k, s in SHAPES.items()}
    if step % 3 == 1:
        gs[NONE_ON] = None
    return gs


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("max_norm", [0.05, 1e3, None], ids=["clip", "noclip", "noclipping"])
def test_reference_matches_torch_optimizers(wd, max_norm):
    """35 float64 steps, warm-up 10, one parameter without a gradient on some steps: p, exp_avg, exp_avg_sq, the norm
    and the learning rate equal torch's to float64 rounding."""
    lay, n, n_decay = _layout()
    gen = torch.Generator().manual_seed(3)
    init = {k: torch.randn(s, generator=gen, dtype=torch.float64) for k, s in SHAPES.items()}
    params = {k: torch.nn.Parameter(v.clone()) for k, v in init.items()}
    opt = OR.reference_optimizer(params.values(), lr=1e-2, wd=wd)
    assert isinstance(opt, torch.optim.Adam if wd == 0 else torch.optim.AdamW)
    sched = torch.optim.lr_scheduler.LinearLR(opt, start_factor=1e-7, end_factor=1.0, total_iters=10)
    p = torch.cat([init[k].reshape(-1) for k in SHAPES])
    m, v, t = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for step in range(35):
        gs = _grads(step, gen, 1.0)
        for k, g in gs.items():
            params[k].grad = g.clone() if g is not None else None
        if max_norm is not None:
            tn = float(torch.nn.utils.clip_grad_norm_(list(params.values()), max_norm))
        frozen = [lay[k] for k, g in gs.items() if g is None]
        gflat = torch.cat([(g if g is not None else torch.zeros(SHAPES[k], dtype=torch.float64)).reshape(-1) for k, g in gs.items()])
        live = OR.live_mask(n, frozen)
        t = t + live.double()
        lr = 1e-2 * OR.lr_factor(step, 10)
        assert abs(opt.param_groups[0]["lr"] - lr) <= 1e-15 * lr
        before, torch_before = p.clone(), params[NONE_ON].detach().clone()
        p, m, v, norm = OR.adamw_update(p, gflat, m, v, t=t, lr=lr, wd=wd, n_decay=n_decay, max_grad_norm=max_norm, frozen=frozen)
        if max_norm is not None:
            assert abs(norm - tn) <= 1e-14 * tn
        opt.step()
        sched.step()
        for k, (a, b) in lay.items():
            assert torch.allclose(p[a:b], params[k].detach().reshape(-1), rtol=1e-13, atol=1e-15), (step, k)
            st = opt.state.get(params[k])
            if st is None:
                assert not bool(m[a:b].any()) and not bool(v[a:b].any())
                continue
            assert torch.allclose(m[a:b], st["exp_avg"].reshape(-1), rtol=1e-12, atol=1e-16), (step, k)
            assert torch.allclose(v[a:b], st["exp_avg_sq"].reshape(-1), rtol=1e-12, atol=1e-18), (step, k)
            assert int(float(st["step"])) == int(t[a])
        # a parameter skipped this step keeps its values exactly
        for a, b in frozen:
            assert torch.equal(p[a:b], before[a:b]) and torch.equal(params[NONE_ON].detach(), torch_before)


@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_reference_matches_restatement(wd):
    """oracle.restatement.clip_and_adamw over 30 steps (clip active on some, a parameter without gradient on others)."""
    lay, n, n_decay = _layout()
    gen = torch.Generator().manual_seed(11)
    init = {k: torch.randn(s, generator=gen, dtype=torch.float64) for k, s in SHAPES.items()}
    params = {k: v.clone() for k, v in init.items()}
    state = {}
    p = torch.cat([init[k].reshape(-1) for k in SHAPES])
    m, v, t = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for step in range(30):
        gs = _grads(step, gen, 0.3 if step % 2 else 3.0)
        norm_r = R.clip_and_adamw(params, gs, state, step=step, lr=1e-2, wd=wd, max_grad_norm=1.0, warmup_iters=10)
        frozen = [lay[k] for k, g in gs.items() if g is None]
        gflat = torch.cat([(g if g is not None else torch.zeros(SHAPES[k], dtype=torch.float64)).reshape(-1) for k, g in gs.items()])
        t = t + OR.live_mask(n, frozen).double()
        p, m, v, norm = OR.adamw_update(p, gflat, m, v, t=t, lr=1e-2 * OR.lr_factor(step, 10), wd=wd, n_decay=n_decay,
                                        max_grad_norm=1.0, frozen=frozen)
        assert abs(norm - norm_r) <= 1e-14 * norm_r
        for k, (a, b) in lay.items():
            assert torch.allclose(p[a:b], params[k].reshape(-1), rtol=1e-13, atol=1e-15), (step, k)
            if k in state:
                assert torch.allclose(m[a:b], state[k]["m"].reshape(-1), rtol=1e-12, atol=1e-16), (step, k)
                assert torch.allclose(v[a:b], state[k]["v"].reshape(-1), rtol=1e-12, atol=1e-18), (step, k)


@pytest.mark.skipif(not ref_harness.available(), reason="needs a reference checkout (OMLM_REFERENCE_ROOT)")
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_reference_optimizer_is_get_optimizer(wd):
    """reference_optimizer builds what the reference's get_optimizer builds: class, groups, hyper-parameters; the state
    files of each load into the other."""
    ref_harness.import_reference()
    ref_opt = importlib.import_module("open_musiclm.optimizer")
    gen = torch.Generator().manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(s, generator=gen)) for s in SHAPES.values()]
    a = ref_opt.get_optimizer(ps, lr=3e-4, wd=wd)
    b = OR.reference_optimizer(ps, lr=3e-4, wd=wd)
    assert type(a) is type(b) and len(a.param_groups) == len(b.param_groups)
    for ga, gb in zip(a.param_groups, b.param_groups):
        assert [id(p) for p in ga["params"]] == [id(p) for p in gb["params"]]
        assert {k: v for k, v in ga.items() if k != "params"} == {k: v for k, v in gb.items() if k != "params"}
    for p in ps:
        p.grad = torch.ones_like(p)
    a.step()
    b.load_state_dict(a.state_dict())
    a.load_state_dict(b.state_dict())
    sa = ref_opt.get_linear_scheduler(a, total_iters=10)
    sb = torch.optim.lr_scheduler.LinearLR(b, start_factor=1e-7, end_factor=1.0, total_iters=10)
    assert sa.state_dict() == sb.state_dict()


def test_lr_factor_is_linear_lr():
    for warmup in (1, 5, 10, 6000):
        opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1, dtype=torch.float64))], lr=3e-4)
        sched = torch.optim.lr_scheduler.LinearLR(opt, start_factor=1e-7, end_factor=1.0, total_iters=warmup)
        for s in range(min(warmup + 3, 40)):
            want = opt.param_groups[0]["lr"]
            assert abs(3e-4 * OR.lr_factor(s, warmup) - want) <= 1e-14 * want, (warmup, s)
            opt.step()
            sched.step()
    assert OR.lr_factor(0, 10) == 1e-7 and OR.lr_factor(7, 0) == 1.0


# ------------------------------------------------------------------------------------------------ error scales
def adamw_replica(p, g, m, v, n_decay, hyper, sumsq, rsqrt_ulps=0, mutation=None):
    """adamw_kernel in numpy float32, one IEEE rounding per operation; rsqrtf's result moved by rsqrt_ulps ulps.
    mutation: one of the wrong variants the scales must reject."""
    f = np.float32
    p, g, m, v = (x.numpy().astype(np.float32) for x in (p, g, m, v))
    lr, b1, b2, eps, wd, bc1, bc2, max_norm, pre = (f(x) for x in hyper)
    coef = pre
    if max_norm > 0:
        norm = f(math.sqrt(sumsq))
        coef = f(coef * min(f(1), f(max_norm / f(norm + (f(0) if mutation == "clip_no_eps" else f(1e-6))))))
    step = f(lr / bc1)
    inv = f(1.0 / math.sqrt(float(bc2)))
    for _ in range(abs(rsqrt_ulps)):
        inv = np.nextafter(inv, f(np.inf) if rsqrt_ulps > 0 else f(0))
    decay = f(f(1) - f(lr * wd))
    gi = g * coef
    idx = np.arange(p.size)
    pi = np.where(idx < (p.size if mutation == "decay_all" else n_decay), p * decay, p)
    mi = b1 * m + (f(1) - b1) * gi
    vi = b2 * v + (f(1) - b2) * gi * gi
    denom = np.sqrt(vi + eps) * inv if mutation == "eps_in_sqrt" else np.sqrt(vi) * inv + eps
    return pi - step * (mi / denom), mi, vi


CASES = [dict(t=1, fac=1e-7, wd=0.01, max_norm=0.5), dict(t=2, fac=0.3, wd=0.0, max_norm=1e6), dict(t=10, fac=1.0, wd=0.01, max_norm=None),
         dict(t=1000, fac=1.0, wd=0.01, max_norm=1e-4, prescale=1 / 3, gscale=1e-8), dict(t=100000, fac=1.0, wd=0.01, max_norm=0.5, prescale=0.125)]


def _check(case, n=20011, rsqrt_ulps=0, mutation=None, t_shift=0, fac_shift=None):
    p, g, m, v = OR.adamw_cases(n, seed=case["t"])
    g = g * case.get("gscale", 1.0)
    n_decay = n // 3
    pre = case.get("prescale", 1.0)
    kw = dict(t=case["t"], lr=3e-4 * case["fac"], wd=case["wd"], n_decay=n_decay, max_grad_norm=case["max_norm"], prescale=pre)
    S = OR.sumsq(g, pre)
    hk = dict(kw, t=case["t"] - t_shift, lr=3e-4 * (fac_shift if fac_shift is not None else case["fac"]))
    hk.pop("n_decay")
    hyper = OR.hyper_vector(t=hk["t"], lr=hk["lr"], wd=hk["wd"], max_grad_norm=hk["max_grad_norm"], prescale=pre)
    got = adamw_replica(p, g, m, v, n_decay, hyper, S, rsqrt_ulps, mutation)
    want = OR.adamw_update(p, g, m, v, **kw)[:3]
    bound = OR.adamw_bound(p, g, m, v, **kw, sumsq_value=S)
    return [float(((torch.from_numpy(x.astype(np.float64)) - w).abs() / b.clamp_min(1e-300)).max()) for x, w, b in zip(got, want, bound)]


@pytest.mark.parametrize("case", CASES, ids=[f"t{c['t']}" for c in CASES])
def test_adamw_scales_bound_an_fp32_replica(case):
    """The per-element scales hold for an fp32 replica of the kernel, also with rsqrtf off by its full 2 ulp either way;
    wrong variants of the arithmetic leave them."""
    for ulps in (0, 2, -2):
        worst = _check(case, rsqrt_ulps=ulps)
        assert max(worst) <= 1.0, (ulps, worst)
    assert _check(case, mutation="eps_in_sqrt")[0] > 1.0
    if case["wd"] > 0 and case["fac"] == 1.0:
        assert _check(case, mutation="decay_all")[0] > 1.0
    if case["t"] in (2, 10):
        assert _check(case, t_shift=1)[0] > 1.0                    # bias corrections from t - 1
    if case["max_norm"] == 1e-4:
        assert _check(case, mutation="clip_no_eps")[0] > 1.0
    if case["fac"] == 1e-7:
        assert _check(case, fac_shift=OR.lr_factor(1, 10))[0] > 1.0  # warm-up factor one step ahead


def sumsq_replica(g, blocks, threads=512, drop_tail=False):
    """sumsq_kernel in numpy float32: per-thread chains over the grid stride, the tail in thread 0, pairwise fp32 sums
    over each block, the blocks' sums in float64."""
    x = g.numpy().astype(np.float32)
    n = x.size
    n4 = n // 4
    T = blocks * threads
    q = x[:4 * n4].reshape(n4, 4)
    q2 = q * q
    sq = ((q2[:, 0] + q2[:, 1]) + q2[:, 2]) + q2[:, 3]
    s = np.zeros(T, dtype=np.float32)
    for i0 in range(0, n4, T):
        part = sq[i0:i0 + T]
        s[:part.size] += part
    if not drop_tail:
        for j in range(n & 3):
            s[j] += x[4 * n4 + j] * x[4 * n4 + j]
    s = s.reshape(blocks, threads)
    while s.shape[1] > 1:
        s = s[:, 0::2] + s[:, 1::2]
    return float(s[:, 0].astype(np.float64).sum())


@pytest.mark.parametrize("n", [1, 2, 3, 7, 4097, 3 * 512 * 4 * 5 + 3])
@pytest.mark.parametrize("scale", [1e-20, 1.0, 1e15])
def test_sumsq_scale_bounds_an_fp32_replica(n, scale):
    gen = torch.Generator().manual_seed(n)
    g = (torch.randn(n, generator=gen) * scale).float()
    blocks = 3
    S = OR.sumsq(g)
    b = OR.sumsq_bound(g, 1.0, blocks)
    assert abs(sumsq_replica(g, blocks) - S) <= b
    if n & 3 and S > 0:
        tail = float(g[-(n & 3):].double().square().sum())
        if tail > 2 * b:
            assert abs(sumsq_replica(g, blocks, drop_tail=True) - S) > b


# ------------------------------------------------------------------------------------------------ frozen parameters
@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_frozen_parameters_are_the_fixtures_none_gradients(path):
    from open_musiclm_b200.trainer import frozen_parameter_names
    fx = torch.load(path, weights_only=False)
    names = [k for k in fx["state_dict"] if k in fx["grads"]]
    assert frozen_parameter_names(names, fx["ce_weights"]) == {k for k, g in fx["grads"].items() if g is None}


def test_live_ranges():
    from open_musiclm_b200.trainer import live_ranges
    assert live_ranges(10, []) == [(0, 10)]
    assert live_ranges(10, [(0, 10)]) == []
    assert live_ranges(100, [(40, 50), (10, 20), (20, 30)]) == [(0, 10), (30, 40), (50, 100)]
    assert live_ranges(100, [(90, 100)]) == [(0, 90)]

"""The compact form of tests/golden/cbsize_*.pt (recorded by tools/make_golden_codebooks.py), shared by the recorder and
the tests.

A fixture holds no weights: the model is rebuilt from the package's factory under torch.manual_seed(0) (the same
parameter init as the reference's, tests/test_boundary_cpu.py) with the perturbation of oracle/make_golden.py, and
the fixture's SHA-256 of the reference's state dict pins the result.  Large tensors (logits, gradients, parameters after
the optimiser steps) are kept as seeded samples of their entries -- half drawn from the nonzero entries, half from all --
plus their full L2 norm.  The generation fixtures keep the SHA-256 of the Gumbel-noise draws instead of the draws:
they are regenerated from the seed the reference ran under."""
import hashlib

import torch

FULL_MAX = 1024          # tensors up to this many entries are stored whole
HALF = 512               # otherwise: 512 nonzero entries + 512 entries of any value


def state_sha(sd) -> str:
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(v.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def tensor_sha(t) -> str:
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def perturb_(model):
    """oracle/make_golden.py's perturbation of the unit-initialised gammas and q / k scales."""
    g0 = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for k, p in model.named_parameters():
            if k.endswith("gamma") or k.endswith("q_scale") or k.endswith("k_scale"):
                p.mul_(1.0 + 0.2 * torch.randn(p.shape, generator=g0))
    return model


def model_of(fx):
    """The fixture's model on the CPU, rebuilt with this package's factory; checked against the recorded SHA-256."""
    import open_musiclm_b200 as O
    fn = {"semantic": O.create_semantic_transformer, "coarse": O.create_coarse_transformer,
          "fine": O.create_fine_transformer}[fx["stage"]]
    torch.manual_seed(0)
    m = perturb_(fn(**fx["kwargs"]))
    assert state_sha(m.state_dict()) == fx["state_sha"], "rebuilt weights differ from the reference's"
    return m


def sample(t, seed=0):
    """dict(shape, idx int32, val, norm) of tensor t (see the module docstring)."""
    flat = t.detach().reshape(-1).float()
    n = flat.numel()
    if n <= FULL_MAX:
        idx = torch.arange(n)
    else:
        g = torch.Generator().manual_seed(seed)
        nz = flat.nonzero()[:, 0]
        idx = torch.unique(torch.cat([nz[torch.randperm(nz.numel(), generator=g)[:HALF]], torch.randperm(n, generator=g)[:HALF]]))
    return dict(shape=tuple(t.shape), idx=idx.int(), val=flat[idx].clone(), norm=float(flat.double().norm()))


def at(t, s):
    """The entries of tensor t (any device) at the sample's positions, on the CPU."""
    assert tuple(t.shape) == tuple(s["shape"]), (tuple(t.shape), s["shape"])
    return t.detach().reshape(-1)[s["idx"].long().to(t.device)].float().cpu()


def rel_to(t, s):
    """Relative L2 error of t against the sample over its positions."""
    a, b = at(t, s).double(), s["val"].double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def norm_rel(t, s):
    return abs(float(t.detach().double().norm()) - s["norm"]) / max(s["norm"], 1e-30)


def uniforms(fx):
    """The Gumbel-noise draws the reference's generate consumed: torch.zeros(B, C).uniform_(0, 1) per sampled token from
    the CPU generator seeded with fx["noise_seed"]."""
    g = torch.Generator().manual_seed(fx["noise_seed"])
    n, B, C = fx["noise_shape"]
    u = torch.stack([torch.zeros(B, C).uniform_(0, 1, generator=g) for _ in range(n)])
    assert tensor_sha(u) == fx["noise_sha"], "regenerated noise differs from the reference's"
    return u

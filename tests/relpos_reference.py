"""The continuous relative-position-bias MLP (RelativePositionBias, transformer.py:36-67) in float64, shared by
tests/test_relpos_bias_cpu.py and tests/test_relpos_bias_gpu.py.

The MLP maps a distance x to h head biases:  a_0 = silu(W_0 x + b_0),  a_j = silu(W_j a_{j-1} + b_j) for j = 1, 2,
y = W_3 a_2 + b_3.  It is evaluated here on the causal distances 0..N-1, the rows of the engine's table[h, delta].

  table(params, N)        -> [h, N] float64
  grads(params, N, dT)    -> the 8 parameter gradients of sum(table * dT), by float64 autograd
  magnitude(params, N, dT) -> componentwise scales S of the same tensors: every pass repeated with |W|, |b|, |x|, each
                             SiLU replaced by a bound on its magnitude and slope.  An fp32 or bf16x3 evaluation errs by
                             at most a few units of its rounding unit times S, entry by entry.

params: {short name: tensor} with the short names of KEYS (any dtype, any device; everything is promoted to float64)."""
import torch

PREFIX = "transformer.rel_pos_bias."
KEYS = ["net.0.0.weight", "net.0.0.bias", "net.1.0.weight", "net.1.0.bias", "net.2.0.weight", "net.2.0.bias",
        "net.3.weight", "net.3.bias"]
SILU_SLOPE = 1.1        # max |silu'(z)| = 1.0998 (at z = 2.40); also |silu(z)| <= |z|
SILU_CURVE = 0.5        # max |silu''(z)| = 0.5 (at z = 0)


def params_of(sd):
    """The 8 MLP tensors of a state dict or of the engine's parameter views, as float64 copies on the same device."""
    return {k: sd[PREFIX + k].detach().double().clone() for k in KEYS}


def _w(p, j):
    return (p["net.3.weight"], p["net.3.bias"]) if j == 3 else (p[f"net.{j}.0.weight"], p[f"net.{j}.0.bias"])


def distances(N, device="cpu"):
    return torch.arange(N, dtype=torch.float64, device=device)[:, None]


def layers(params, N):
    """The forward pass -> (z [3 x [N, Hr]], a [3 x [N, Hr]], table [h, N]), all float64."""
    x = distances(N, params["net.0.0.weight"].device)
    zs, acts = [], []
    for j in range(3):
        w, b = _w(params, j)
        z = x @ w.t() + b
        x = torch.nn.functional.silu(z)
        zs.append(z)
        acts.append(x)
    w, b = _w(params, 3)
    return zs, acts, (x @ w.t() + b).t()


def table(params, N):
    return layers(params, N)[2]


def bias_table(sd, N, bias_type, heads):
    """table[h, delta] of any bias type from a state dict.  't5': the bucket embedding is looked up with i - j negated
    and clamped at 0 (transformer.py:86-104), so every causal distance reads bucket 0; 'none': no bias."""
    if bias_type == "none":
        return torch.zeros(heads, N, dtype=torch.float64)
    if bias_type == "t5":
        w = sd[PREFIX + "relative_attention_bias.weight"].detach().double()          # [32 buckets, h]
        return w[0][:, None].expand(heads, N).contiguous()
    return table(params_of(sd), N)


def grads(params, N, dT):
    """d sum(table * dT) / d params -> {short name: float64 tensor}."""
    leaves = {k: v.detach().double().clone().requires_grad_(True) for k, v in params.items()}
    with torch.enable_grad():
        t = table(leaves, N)
        t.backward(dT.double())
    return {k: leaves[k].grad for k in KEYS}


def magnitude(params, N, dT=None):
    """Componentwise scales (see the module docstring) -> dict with z / a [3 x [N, Hr]] and table [h, N] and, given
    dT, the 8 gradient scales under the short names of KEYS and dz [3 x [N, Hr]].

    Forward: S_z_j = |W_j| S_a_{j-1} + |b_j| (S_a_{-1} = x), S_a_j = SILU_SLOPE S_z_j, S_table = |W_3| S_a_2 + |b_3|.
    Backward: S_da_2 = |dT|^T |W_3|; an error dz in z moves silu'(z) by up to SILU_CURVE |dz|, so
    S_dz_j = S_da_j (SILU_SLOPE + SILU_CURVE S_z_j); S_dW_j = S_dz_j^T S_a_{j-1}, S_db_j = colsum S_dz_j,
    S_da_{j-1} = S_dz_j |W_j|."""
    ab = {k: v.detach().double().abs() for k, v in params.items()}
    x = distances(N, ab["net.0.0.weight"].device)
    s_in, s_z, s_a = [x], [], []
    for j in range(3):
        w, b = _w(ab, j)
        z = s_in[-1] @ w.t() + b
        s_z.append(z)
        s_a.append(SILU_SLOPE * z)
        s_in.append(s_a[-1])
    w3, b3 = _w(ab, 3)
    out = {"z": s_z, "a": s_a, "table": (s_a[2] @ w3.t() + b3).t()}
    if dT is None:
        return out
    adT = dT.detach().double().abs().to(x.device)                 # [h, N]
    out["net.3.weight"] = adT @ s_a[2]
    out["net.3.bias"] = adT.sum(1)
    s_da = adT.t() @ w3                                             # [N, Hr]
    s_dz = [None] * 3
    for j in (2, 1, 0):
        s_dz[j] = s_da * (SILU_SLOPE + SILU_CURVE * s_z[j])
        w, _ = _w(ab, j)
        out[f"net.{j}.0.weight"] = s_dz[j].t() @ s_in[j]
        out[f"net.{j}.0.bias"] = s_dz[j].sum(0)
        s_da = s_dz[j] @ w
    out["dz"] = s_dz
    return out
